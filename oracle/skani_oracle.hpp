// ============================================================================
// skani_oracle.hpp -- TEST INFRASTRUCTURE ONLY (CPU oracle / CPU baseline).
//
// A C++17 restatement of the ANI hot path of bluenote-1577/skani v0.3.0 (reference
// commit c57dbe7).  The Rust reference cannot be compiled in this environment (no
// cargo/rustc), so this file re-expresses the reference *algorithm*; every function
// cites the reference file:line it follows.  Third-party behaviour the results depend
// on (partitions 0.2.4 PartitionVec, bio 1.4.0 IntervalTree, intervallum 1.4.0
// IntervalSet, fastrand 1.9.0 WyRand, gbdt 0.1.1 predict, needletail 0.5.1 record
// splitting) is restated from the published algorithms and pinned by the reference's
// own golden outputs (see tests/test_oracle_goldens.py, SURVEY.md section 8c).
//
// Nothing in the shipped product (skani_b200/) may include, link or call this code.
// Only tests/, __graft_entry__.smoke() and bench.py's cpu_baseline / --impl reference
// legs use it, and only as the checker / CPU baseline.
// ============================================================================
#pragma once
#include <cstdint>
#include <cstddef>
#include <string>
#include <vector>

namespace orc {

// ---- constants: src/params.rs:6-62 -----------------------------------------------------------
constexpr int K_MARKER_DNA = 21;            // params.rs:35
constexpr uint32_t CHUNK_SIZE_DNA = 20000;  // params.rs:40
constexpr size_t MIN_LENGTH_CONTIG = 500;   // params.rs:42
constexpr uint32_t MIN_LENGTH_COVER = 500;  // params.rs:44
constexpr uint32_t BP_CHAIN_BAND = 2500;    // params.rs:45
constexpr double D_MAX_GAP_LENGTH = 300.;   // params.rs:19
constexpr double D_MAX_LIN_LENGTH = 5000.;  // params.rs:21
constexpr double D_ANCHOR_SCORE_ANI = 20.;  // params.rs:22
constexpr size_t D_MIN_ANCHORS_ANI = 3;     // params.rs:24
constexpr double SEARCH_ANI_CUTOFF_DEFAULT = 0.80;  // params.rs:48
constexpr size_t SCREEN_MINIMUM_KMERS = 20;         // params.rs:49
constexpr float OVERLAP_ORTHOLOGOUS_FRACTION = 0.50f;  // params.rs:52
constexpr uint32_t TOTAL_BASES_REGRESS_CUTOFF = 150000;  // params.rs:53

// ---- types.rs -----------------------------------------------------------------------------------
uint64_t mm_hash64(uint64_t key);           // types.rs:86-96
extern const uint8_t* const BYTE_TO_SEQ;    // types.rs:40-49 (256 entries)

struct SeedPosition {                       // types.rs:125-192
  uint32_t pos;
  uint32_t contig_index_canonical;          // contig<<1 | canonical
  bool canonical() const { return contig_index_canonical & 1u; }
  uint32_t contig_index() const { return contig_index_canonical >> 1; }
};

// Open-addressing stand-ins for the reference's hashbrown maps (types.rs:56-69). Iteration order is
// arbitrary in both; no result depends on it (SURVEY App. A.5).
class KmerSeeds {  // HashMap<u32,u64> keyed by seed k-mer, value = TaggedIndex (types.rs:207-244)
 public:
  KmerSeeds();
  uint64_t* find(uint32_t key);
  const uint64_t* find(uint32_t key) const;
  void insert(uint32_t key, uint64_t val);  // key must be absent
  size_t size() const { return n_; }
  // iteration
  size_t capacity() const { return keys_.size(); }
  bool slot_used(size_t s) const { return used_[s]; }
  uint32_t slot_key(size_t s) const { return keys_[s]; }
  uint64_t slot_val(size_t s) const { return vals_[s]; }
 private:
  void grow();
  std::vector<uint32_t> keys_;
  std::vector<uint64_t> vals_;
  std::vector<uint8_t> used_;
  size_t n_ = 0, mask_ = 0;
};

class MarkerSet {  // HashSet<u64> (types.rs:68, 269)
 public:
  MarkerSet();
  bool contains(uint64_t key) const;
  void insert(uint64_t key);
  size_t size() const { return n_; }
  size_t capacity() const { return keys_.size(); }
  bool slot_used(size_t s) const { return keys_[s] != EMPTY; }
  uint64_t slot_key(size_t s) const { return keys_[s]; }
 private:
  static constexpr uint64_t EMPTY = ~0ull;  // markers are < 2^42
  void grow();
  std::vector<uint64_t> keys_;
  size_t n_ = 0, mask_ = 0;
};

struct SketchParams {  // params.rs:137-146 (AAI members omitted: out of scope)
  uint64_t c = 125, k = 15, marker_c = 1000;
};

struct Sketch {  // types.rs:253-277
  std::string file_name;
  bool has_seeds = false;  // kmer_seeds_k.is_some()
  KmerSeeds kmer_seeds_k;
  std::vector<std::vector<SeedPosition>> multi_position_storage;
  std::vector<std::string> contigs;
  uint64_t total_sequence_length = 0;
  std::vector<uint32_t> contig_lengths;
  MarkerSet marker_seeds;
  uint64_t marker_c = 0, c = 0, k = 0;
  uint64_t contig_order = 0;
  bool individual_contig = false;

  void add_seed_position(uint32_t seed, SeedPosition p);                 // types.rs:281-304
  // returns count; *out points at the positions (valid until next call on this thread for singles)
  size_t get_seed_positions(uint32_t seed, const SeedPosition** out, SeedPosition* tmp) const;  // types.rs:306-320
};

// seeding.rs:225-323 (scalar) and avx2_seeding.rs:33-272 (the path taken on x86-64 with AVX2; authoritative)
void fmh_seeds_scalar(const uint8_t* s, size_t n, const SketchParams& sp, uint32_t contig_index, Sketch& sk);
void fmh_seeds_avx2sem(const uint8_t* s, size_t n, const SketchParams& sp, uint32_t contig_index, Sketch& sk);
void set_avx2_intrinsics(bool on);   // baseline only: run the 4-lane AVX2 instruction mix of avx2_seeding.rs instead of the lane-by-lane form
bool avx2_intrinsics();

// file_io.rs:141-252 / 253-362.  Returns sketches sorted by (file_name, contig_order).
// warnings (one per skipped file) are appended to *warn if non-null.
std::vector<Sketch> fastx_to_sketches(const std::vector<std::string>& files, const SketchParams& sp,
                                      bool individual_contig, bool use_avx2_semantics, int threads,
                                      std::vector<std::string>* warn);
// In-memory variant of the same assembly rules (contigs already split; names optional).
Sketch sketch_from_contigs(const std::string& file_name, const std::vector<std::pair<const uint8_t*, size_t>>& contigs,
                           const std::vector<std::string>* names, const SketchParams& sp, bool use_avx2_semantics);

// ---- screen.rs --------------------------------------------------------------------------------------
struct KmerToSketch;  // inverted index marker -> sketch ids (screen.rs:190-210)
KmerToSketch* kmer_to_sketch_from_refs(const std::vector<const Sketch*>& refs);
void kmer_to_sketch_free(KmerToSketch*);
// screen.rs:148-189; returns ascending ids
std::vector<uint32_t> screen_refs(double identity, const KmerToSketch& idx, const Sketch& q,
                                  const std::vector<const Sketch*>& refs, bool rescue_small);
// screen.rs:39-77
std::vector<uint32_t> screen_refs_indices(double identity, const KmerToSketch& idx, const Sketch& q,
                                          const std::vector<const Sketch*>& refs);
// screen.rs:84-142
bool check_markers_quickly(const Sketch& ref, const Sketch& query, double screen_val, bool rescue_small);

// ---- chain.rs ---------------------------------------------------------------------------------------
struct CommandParams {  // subset of params.rs:96-123 that reaches the hot path
  double screen_val = 0.;
  bool robust = false, median = false;
  double min_aligned_frac = 0.15, both_min_aligned_frac = -0.01;  // after /100 (parse.rs)
  bool learned_ani = true;
  bool rescue_small = true;
};

struct MapParams {  // params.rs:75-93
  uint32_t fragment_length;
  double max_gap_length, anchor_score;
  size_t min_anchors;
  double frac_cover_cutoff, both_frac_cover_cutoff;
  size_t index_chain_band;
  size_t k;
  double min_score;
  bool robust, median;
  uint32_t bp_chain_band, min_length_cover;
  int model;  // -1 none, 0 = C125, 1 = C200 (regression.rs:12-28)
};

struct Anchor {  // types.rs:499-506; derived Ord = field order
  uint32_t query_contig, query_pos, ref_contig, ref_pos;
  bool reverse_match;
};

struct ChainInterval {  // types.rs:508-519
  double score;
  size_t num_anchors;
  uint32_t q0, q1, r0, r1;
  size_t ref_contig, query_contig, chunk_id;
  bool reverse_chain;
  uint32_t overlap;
};

struct AniEstResult {  // types.rs:559-582 (strings resolved by the caller from the sketches)
  float ani = 0, align_fraction_query = 0, align_fraction_ref = 0;
  float ci_upper = 0, ci_lower = 0;
  float quant_90_contig_len_q = 0, quant_90_contig_len_r = 0, quant_50_contig_len_q = 0,
        quant_50_contig_len_r = 0, quant_10_contig_len_q = 0, quant_10_contig_len_r = 0;
  float std = 0;
  uint32_t num_contigs_q = 0, num_contigs_r = 0, avg_chain_int_len = 0, total_bases_covered = 0;
};

struct ChainDebug {  // parity taps (not in the reference): intermediate products of chain_seeds
  bool switched = false;
  std::vector<Anchor> anchors;                 // sorted (chain.rs:721)
  std::vector<uint32_t> chunk_first;           // first anchor index of every chunk (+ sentinel = n anchors)
  std::vector<uint32_t> chunk_nseeds;          // |seeds_in_chunk[i]|
  std::vector<double> score;                   // per anchor (chain.rs:881)
  std::vector<uint32_t> pointer;               // per anchor, chunk-local index (chain.rs:882)
  std::vector<ChainInterval> intervals_all;    // after the descending sort (chain.rs:1012)
  std::vector<uint8_t> interval_kept;          // greedy decision per sorted interval
  std::vector<std::pair<double, size_t>> ani_ests;  // sorted (est, weight) (chain.rs:414)
  std::vector<uint32_t> chunk_stats;           // 9 per chunk: the fields of ChunkStats up to `filtered`
};

// one chunk of calculate_ani (chain.rs:204-394): the kept intervals' sums, the seed counts and the chunk's identity.  The seed
// counts are taken for every chunk with an interval (the reference counts them only for chunks that pass :253-259).
struct ChunkStats {
  size_t total_anchors = 0;
  uint32_t rq0 = UINT32_MAX, rq1 = 0;   // total_range_query
  uint32_t tbcq = 0;                    // total_bases_contained_query (wrapping u32)
  uint32_t n_int = 0;
  size_t n_seeds = 0, num_in = 0, upper_lower = 0;
  bool filtered = false;                // the putative-ANI filter replaced n_seeds by upper_lower (:336-347)
  bool valid = false;                   // the chunk yields an estimate
  double est = 0.;
  size_t weight = 0;
};
uint32_t padded_start(uint32_t q0, uint32_t c);  // chain.rs:239-240, i32 arithmetic wrapping as in a release build
// filtered / valid / est / weight from the other fields
void chunk_estimate(ChunkStats& s, uint32_t c, size_t k, uint32_t min_length_cover);
ChunkStats chunk_stats(const std::vector<ChainInterval>& intervals, const std::vector<uint32_t>& seeds, uint32_t c, size_t k,
                       uint32_t min_length_cover, bool switched);

// chain_anchors_ani + get_chain_intervals (chain.rs:838-1007) on given chunks, each sorted as get_anchors leaves it
// (chain.rs:721): the chain intervals of every chunk (chunk_id = its index) in emission order, and optionally the DP's score
// and chunk-local pointer of every anchor, chunk after chunk
std::vector<ChainInterval> chain_chunks(const std::vector<std::vector<Anchor>>& chunks, const MapParams& mp,
                                        std::vector<double>* score = nullptr, std::vector<uint32_t>* pointer = nullptr);
// get_nonoverlapping_chains (chain.rs:1008-1099): sorts `intervals` into the descending order of :1012 and returns the kept
// ones per chunk.  Optionally per sorted interval: kept (0 / 1), and hits = 2 per interval, the number of kept intervals its
// ref / query range overlaps (the IntervalTree::find counts of :1029, :1059)
std::vector<std::vector<ChainInterval>> get_nonoverlapping_chains(std::vector<ChainInterval>& intervals, size_t num_chunks,
                                                                  std::vector<uint8_t>* kept = nullptr,
                                                                  std::vector<uint32_t>* hits = nullptr);
// the kept intervals' summed (q1 - q0) - overlap + 2c + k (wrapping u32) and their number: avg_chain_int_len = sum / n
// (chain.rs:244-249, :421)
void chain_len_sums(const std::vector<std::vector<ChainInterval>>& int_chunks, uint32_t c, size_t k, uint32_t* sum,
                    uint32_t* n);

int get_model_id(uint64_t c, bool learned_ani);  // regression.rs:12-28
MapParams map_params_from_sketch(const Sketch& ref, const CommandParams& cp, int model);  // chain.rs:88-142
AniEstResult chain_seeds(const Sketch& ref, const Sketch& query, const MapParams& mp, ChainDebug* dbg = nullptr);  // chain.rs:144-171
float gbdt_predict(int model, const float x[5]);  // gbdt 0.1.1 GBDT::predict, LAD
// the tail of calculate_ani plus predict_from_ani_res (chain.rs:422-555, regression.rs:30-64): trimmed weighted mean, std,
// bootstrap CI, AF cutoffs and learned ANI (mp.model >= 0) from the sorted (est, weight) list; quantiles are {q10, q50, q90}
// of each genome's contig lengths.  An empty list gives ani = NaN.  num_contigs_* are left 0 for the caller.
AniEstResult final_estimate(const std::vector<std::pair<double, size_t>>& ani_ests, uint32_t total_query_bases,
                            uint32_t avg_chain_int_len, uint64_t query_total_len, uint64_t ref_total_len,
                            const float quant_q[3], const float quant_r[3], const MapParams& mp);

// ---- drivers (pair loops of triangle.rs:71-105 / dist.rs:98-144 / search.rs:119-247) -------------
struct PairResult { uint32_t ref_id, query_id; AniEstResult r; };
std::vector<PairResult> triangle(const std::vector<const Sketch*>& sk, const CommandParams& cp, int threads,
                                 uint64_t* n_chained = nullptr, double* t_screen = nullptr, double* t_chain = nullptr);
std::vector<PairResult> dist(const std::vector<const Sketch*>& refs, const std::vector<const Sketch*>& queries,
                             const CommandParams& cp, bool use_index, int threads);
std::vector<PairResult> search(const std::vector<const Sketch*>& refs, const std::vector<const Sketch*>& queries,
                               const CommandParams& cp, bool use_index, int threads);

}  // namespace orc
