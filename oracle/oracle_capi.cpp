// ============================================================================
// oracle_capi.cpp -- TEST INFRASTRUCTURE ONLY.  C entry points over skani_oracle.cpp
// for the Python test-suite / bench CPU-baseline leg (ctypes).  Not part of the product.
// ============================================================================
#include <cstring>
#include <cstdlib>
#include <chrono>
#include <algorithm>
#include <malloc.h>

#include "skani_oracle.hpp"

// The CPU baseline should not be handicapped by glibc malloc defaults under 100+ threads: multi-100 KB vectors would be
// mmap'ed/munmap'ed on every pair (serialising on the process' mm lock).  Keep them on the per-thread arenas instead.
namespace {
struct MallocTuning {
  MallocTuning() {
    mallopt(M_MMAP_THRESHOLD, 512 << 20);
    mallopt(M_TRIM_THRESHOLD, 1 << 30);
    mallopt(M_ARENA_MAX, 512);
  }
} g_malloc_tuning;
}  // namespace

using namespace orc;

extern "C" {

struct orc_result {  // same field order as sk_ani_result in include/skani_b200.h
  float ani, af_query, af_ref, ci_lower, ci_upper, std;
  float q90_q, q90_r, q50_q, q50_r, q10_q, q10_r;
  uint32_t num_contigs_q, num_contigs_r, avg_chain_int_len, total_bases_covered;
  uint32_t ref_id, query_id;
};

struct orc_cmd {
  double screen_val, min_aligned_frac, both_min_aligned_frac;
  int32_t robust, median, learned_ani, rescue_small;
};

static CommandParams to_cp(const orc_cmd* c) {
  CommandParams cp;
  cp.screen_val = c->screen_val;
  cp.min_aligned_frac = c->min_aligned_frac;
  cp.both_min_aligned_frac = c->both_min_aligned_frac;
  cp.robust = c->robust; cp.median = c->median; cp.learned_ani = c->learned_ani; cp.rescue_small = c->rescue_small;
  return cp;
}
static void to_res(const AniEstResult& a, uint32_t rid, uint32_t qid, orc_result* o) {
  o->ani = a.ani; o->af_query = a.align_fraction_query; o->af_ref = a.align_fraction_ref;
  o->ci_lower = a.ci_lower; o->ci_upper = a.ci_upper; o->std = a.std;
  o->q90_q = a.quant_90_contig_len_q; o->q90_r = a.quant_90_contig_len_r;
  o->q50_q = a.quant_50_contig_len_q; o->q50_r = a.quant_50_contig_len_r;
  o->q10_q = a.quant_10_contig_len_q; o->q10_r = a.quant_10_contig_len_r;
  o->num_contigs_q = a.num_contigs_q; o->num_contigs_r = a.num_contigs_r;
  o->avg_chain_int_len = a.avg_chain_int_len; o->total_bases_covered = a.total_bases_covered;
  o->ref_id = rid; o->query_id = qid;
}

uint64_t orc_mm_hash64(uint64_t x) { return mm_hash64(x); }
int orc_set_avx2_intrinsics(int on) { set_avx2_intrinsics(on != 0); return avx2_intrinsics() ? 1 : 0; }

// ---- sketching ------------------------------------------------------------------------------------
// Sketch every file; returns a malloc'd array of handles in (file_name, contig_order) order.
int orc_sketch_files(const char** paths, int n, uint64_t c, uint64_t k, uint64_t marker_c, int individual,
                     int avx2sem, int threads, void*** out, int* n_out, int* n_warn) {
  std::vector<std::string> files(paths, paths + n);
  SketchParams sp; sp.c = c; sp.k = k; sp.marker_c = marker_c;
  if (c > marker_c) return -1;  // params.rs:183-185 (reference panics)
  std::vector<std::string> warn;
  std::vector<Sketch> v = fastx_to_sketches(files, sp, individual != 0, avx2sem != 0, threads, &warn);
  void** arr = (void**)malloc(sizeof(void*) * (v.size() + 1));
  for (size_t i = 0; i < v.size(); i++) arr[i] = new Sketch(std::move(v[i]));
  *out = arr; *n_out = (int)v.size();
  if (n_warn) *n_warn = (int)warn.size();
  return 0;
}
void orc_free_array(void* p) { free(p); }

// contigs given as one concatenated ASCII buffer + n_contigs+1 offsets
void* orc_sketch_from_contigs(const char* name, const uint8_t* bases, const uint64_t* off, uint32_t n_contigs,
                              uint64_t c, uint64_t k, uint64_t marker_c, int avx2sem) {
  SketchParams sp; sp.c = c; sp.k = k; sp.marker_c = marker_c;
  std::vector<std::pair<const uint8_t*, size_t>> ctgs;
  for (uint32_t i = 0; i < n_contigs; i++) ctgs.push_back({bases + off[i], (size_t)(off[i + 1] - off[i])});
  return new Sketch(sketch_from_contigs(name, ctgs, nullptr, sp, avx2sem != 0));
}
void orc_sketch_free(void* s) { delete (Sketch*)s; }

// time seeding only (CPU baseline leg): seeds n_contigs contigs `reps` times, returns seconds
double orc_time_seeding(const uint8_t* bases, const uint64_t* off, uint32_t n_contigs, uint64_t c, uint64_t k,
                        uint64_t marker_c, int threads) {
  SketchParams sp; sp.c = c; sp.k = k; sp.marker_c = marker_c;
  auto t0 = std::chrono::steady_clock::now();
#pragma omp parallel for schedule(dynamic) num_threads(threads > 0 ? threads : 1)
  for (long i = 0; i < (long)n_contigs; i++) {
    Sketch sk;
    sk.c = c; sk.k = k;
    fmh_seeds_avx2sem(bases + off[i], (size_t)(off[i + 1] - off[i]), sp, 0, sk);
  }
  return std::chrono::duration<double>(std::chrono::steady_clock::now() - t0).count();
}

uint64_t orc_sketch_n_records(void* s) {
  Sketch* sk = (Sketch*)s;
  uint64_t n = 0;
  const KmerSeeds& m = sk->kmer_seeds_k;
  for (size_t i = 0; i < m.capacity(); i++) {
    if (!m.slot_used(i)) continue;
    uint64_t t = m.slot_val(i);
    n += (t & 1) ? 1 : sk->multi_position_storage[(size_t)(t >> 1)].size();
  }
  return n;
}
uint64_t orc_sketch_n_kmers(void* s) { return ((Sketch*)s)->kmer_seeds_k.size(); }
uint64_t orc_sketch_n_markers(void* s) { return ((Sketch*)s)->marker_seeds.size(); }
uint64_t orc_sketch_n_contigs(void* s) { return ((Sketch*)s)->contigs.size(); }
uint64_t orc_sketch_total_len(void* s) { return ((Sketch*)s)->total_sequence_length; }
const char* orc_sketch_file_name(void* s) { return ((Sketch*)s)->file_name.c_str(); }
const char* orc_sketch_contig_name(void* s, uint64_t i) { return ((Sketch*)s)->contigs[i].c_str(); }
uint64_t orc_sketch_contig_order(void* s) { return ((Sketch*)s)->contig_order; }

// export as flat arrays: records sorted by (kmer, contig, pos); markers ascending; contig lengths in order
void orc_sketch_export(void* s, uint32_t* kmer, uint32_t* pos, uint32_t* cc, uint64_t* markers, uint32_t* contig_lengths) {
  Sketch* sk = (Sketch*)s;
  struct Rec { uint32_t kmer, pos, cc; };
  std::vector<Rec> recs;
  const KmerSeeds& m = sk->kmer_seeds_k;
  SeedPosition tmp;
  for (size_t i = 0; i < m.capacity(); i++) {
    if (!m.slot_used(i)) continue;
    const SeedPosition* p;
    size_t n = sk->get_seed_positions(m.slot_key(i), &p, &tmp);
    for (size_t a = 0; a < n; a++) recs.push_back({m.slot_key(i), p[a].pos, p[a].contig_index_canonical});
  }
  std::sort(recs.begin(), recs.end(), [](const Rec& a, const Rec& b) {
    if (a.kmer != b.kmer) return a.kmer < b.kmer;
    if ((a.cc >> 1) != (b.cc >> 1)) return (a.cc >> 1) < (b.cc >> 1);
    if (a.pos != b.pos) return a.pos < b.pos;
    return a.cc < b.cc;
  });
  for (size_t i = 0; i < recs.size(); i++) { kmer[i] = recs[i].kmer; pos[i] = recs[i].pos; cc[i] = recs[i].cc; }
  std::vector<uint64_t> mk;
  const MarkerSet& ms = sk->marker_seeds;
  for (size_t i = 0; i < ms.capacity(); i++) if (ms.slot_used(i)) mk.push_back(ms.slot_key(i));
  std::sort(mk.begin(), mk.end());
  for (size_t i = 0; i < mk.size(); i++) markers[i] = mk[i];
  for (size_t i = 0; i < sk->contig_lengths.size(); i++) contig_lengths[i] = sk->contig_lengths[i];
}

// ---- screen -----------------------------------------------------------------------------------------
int orc_check_markers_quickly(void* ref, void* query, double screen_val, int rescue_small) {
  return check_markers_quickly(*(Sketch*)ref, *(Sketch*)query, screen_val, rescue_small != 0) ? 1 : 0;
}
// rows of the triangle screen: for every i the ascending list of j > i that pass screen_refs(i). CSR output.
int orc_screen_triangle(void** sk, int n, double screen_val, int rescue_small, uint64_t** row_off, uint32_t** cols) {
  std::vector<const Sketch*> v;
  for (int i = 0; i < n; i++) v.push_back((Sketch*)sk[i]);
  double sv = screen_val == 0. ? SEARCH_ANI_CUTOFF_DEFAULT : screen_val;
  KmerToSketch* idx = kmer_to_sketch_from_refs(v);
  std::vector<std::vector<uint32_t>> rows(n);
  for (int i = 0; i + 1 < n; i++) {
    auto pass = screen_refs(sv, *idx, *v[i], v, rescue_small != 0);
    for (uint32_t j : pass) if ((int)j > i) rows[i].push_back(j);
  }
  kmer_to_sketch_free(idx);
  uint64_t* ro = (uint64_t*)malloc(sizeof(uint64_t) * (n + 1));
  uint64_t tot = 0;
  for (int i = 0; i < n; i++) { ro[i] = tot; tot += rows[i].size(); }
  ro[n] = tot;
  uint32_t* cs = (uint32_t*)malloc(sizeof(uint32_t) * (tot + 1));
  for (int i = 0; i < n; i++) memcpy(cs + ro[i], rows[i].data(), rows[i].size() * 4);
  *row_off = ro; *cols = cs;
  return 0;
}
// markers-only sketches (Sketch::get_markers_only): genome g holds markers[mk_off[g] .. mk_off[g+1]), inserted through
// MarkerSet::insert (duplicates collapse as in the reference's HashSet); handles are written to out[0..n)
int orc_sketches_from_markers(int n, const uint64_t* mk_off, const uint64_t* markers, void** out) {
  for (int g = 0; g < n; g++) {
    Sketch* s = new Sketch();
    for (uint64_t i = mk_off[g]; i < mk_off[g + 1]; i++) s->marker_seeds.insert(markers[i]);
    out[g] = s;
  }
  return 0;
}
// query x ref screen as the drivers pick it (orc_dist / orc_search): mode 0 check_markers_quickly(rescue_small), 1 the same
// without rescue, 2 screen_refs, 3 screen_refs_indices.  Output: ascending (ref << 32 | query), malloc'd.
int orc_screen_query_ref(void** refs, int nr, void** queries, int nq, double screen_val, int mode, int rescue_small,
                         uint64_t** pairs, uint64_t* n) {
  if (mode < 0 || mode > 3) return -1;
  std::vector<const Sketch*> r, q;
  for (int i = 0; i < nr; i++) r.push_back((Sketch*)refs[i]);
  for (int i = 0; i < nq; i++) q.push_back((Sketch*)queries[i]);
  const double sv = screen_val == 0. ? SEARCH_ANI_CUTOFF_DEFAULT : screen_val;   // dist.rs:68-77
  std::vector<uint64_t> out;
  if (mode <= 1) {
    const bool rescue = mode == 0 && rescue_small != 0;
    for (int j = 0; j < nq; j++)
      for (int i = 0; i < nr; i++)
        if (check_markers_quickly(*q[j], *r[i], sv, rescue)) out.push_back(((uint64_t)i << 32) | (uint32_t)j);
  } else {
    KmerToSketch* idx = kmer_to_sketch_from_refs(r);
    for (int j = 0; j < nq; j++) {
      auto pass = mode == 3 ? screen_refs_indices(sv, *idx, *q[j], r) : screen_refs(sv, *idx, *q[j], r, rescue_small != 0);
      for (uint32_t i : pass) out.push_back(((uint64_t)i << 32) | (uint32_t)j);
    }
    kmer_to_sketch_free(idx);
  }
  std::sort(out.begin(), out.end());
  uint64_t* o = (uint64_t*)malloc(sizeof(uint64_t) * (out.size() + 1));
  if (!out.empty()) memcpy(o, out.data(), out.size() * 8);
  *pairs = o; *n = out.size();
  return 0;
}

// ---- chain ------------------------------------------------------------------------------------------
int orc_chain(void* ref, void* query, const orc_cmd* cmd, orc_result* out) {
  const Sketch& r = *(Sketch*)ref;
  const Sketch& q = *(Sketch*)query;
  CommandParams cp = to_cp(cmd);
  MapParams mp = map_params_from_sketch(r, cp, get_model_id(r.c, cp.learned_ani));
  to_res(chain_seeds(r, q, mp), 0, 0, out);
  return 0;
}

struct orc_debug {
  ChainDebug d;
  orc_result res;
};
void* orc_chain_debug(void* ref, void* query, const orc_cmd* cmd) {
  const Sketch& r = *(Sketch*)ref;
  const Sketch& q = *(Sketch*)query;
  CommandParams cp = to_cp(cmd);
  MapParams mp = map_params_from_sketch(r, cp, get_model_id(r.c, cp.learned_ani));
  auto* d = new orc_debug();
  to_res(chain_seeds(r, q, mp, &d->d), 0, 0, &d->res);
  return d;
}
void orc_debug_free(void* d) { delete (orc_debug*)d; }
void orc_debug_result(void* d, orc_result* out) { *out = ((orc_debug*)d)->res; }
int orc_debug_switched(void* d) { return ((orc_debug*)d)->d.switched ? 1 : 0; }
uint64_t orc_debug_n_anchors(void* d) { return ((orc_debug*)d)->d.anchors.size(); }
uint64_t orc_debug_n_chunks(void* d) { auto& c = ((orc_debug*)d)->d.chunk_first; return c.empty() ? 0 : c.size() - 1; }
uint64_t orc_debug_n_intervals(void* d) { return ((orc_debug*)d)->d.intervals_all.size(); }
uint64_t orc_debug_n_ests(void* d) { return ((orc_debug*)d)->d.ani_ests.size(); }
// anchors: 5 x u32 per anchor (qcontig,qpos,rcontig,rpos,rev); score i64; pointer u32 (chunk-local)
void orc_debug_anchors(void* dd, uint32_t* a5, int64_t* score, uint32_t* ptr) {
  auto& d = ((orc_debug*)dd)->d;
  for (size_t i = 0; i < d.anchors.size(); i++) {
    const Anchor& a = d.anchors[i];
    a5[5 * i] = a.query_contig; a5[5 * i + 1] = a.query_pos; a5[5 * i + 2] = a.ref_contig; a5[5 * i + 3] = a.ref_pos;
    a5[5 * i + 4] = a.reverse_match;
    score[i] = (int64_t)d.score[i];
    ptr[i] = d.pointer[i];
  }
}
void orc_debug_chunks(void* dd, uint32_t* first /* n_chunks+1 */, uint32_t* nseeds) {
  auto& d = ((orc_debug*)dd)->d;
  for (size_t i = 0; i < d.chunk_first.size(); i++) first[i] = d.chunk_first[i];
  for (size_t i = 0; i < d.chunk_nseeds.size(); i++) nseeds[i] = d.chunk_nseeds[i];
}
// intervals (descending sort order): 11 x i64 per interval: score,num_anchors,q0,q1,r0,r1,ref_contig,query_contig,chunk,rev,kept
void orc_debug_intervals(void* dd, int64_t* f) {
  auto& d = ((orc_debug*)dd)->d;
  for (size_t i = 0; i < d.intervals_all.size(); i++) {
    const ChainInterval& c = d.intervals_all[i];
    int64_t* o = f + 11 * i;
    o[0] = (int64_t)c.score; o[1] = (int64_t)c.num_anchors; o[2] = c.q0; o[3] = c.q1; o[4] = c.r0; o[5] = c.r1;
    o[6] = (int64_t)c.ref_contig; o[7] = (int64_t)c.query_contig; o[8] = (int64_t)c.chunk_id; o[9] = c.reverse_chain;
    o[10] = d.interval_kept[i];
  }
}
// 9 x u32 per chunk: total_anchors, rq0, rq1, tbcq, n_int, n_seeds, num_in, upper_lower, filtered
void orc_debug_chunk_stats(void* dd, uint32_t* out) {
  auto& d = ((orc_debug*)dd)->d;
  if (!d.chunk_stats.empty()) memcpy(out, d.chunk_stats.data(), d.chunk_stats.size() * 4);
}
void orc_debug_ests(void* dd, double* est, uint64_t* weight) {
  auto& d = ((orc_debug*)dd)->d;
  for (size_t i = 0; i < d.ani_ests.size(); i++) { est[i] = d.ani_ests[i].first; weight[i] = d.ani_ests[i].second; }
}

// ---- DP and interval selection on given lists ----------------------------------------------------------------------------
// Shared tail of orc_chain_chunks / orc_select_intervals: the selection of chain.rs:1008-1099 over `good`, written out as
// 11 x i64 per sorted interval (the orc_debug_intervals fields) plus 2 x u32 hits (ref, query: kept intervals overlapping
// it), 5 x u32 per chunk (total_anchors, rq0, rq1, tbcq, n_int of the kept intervals, chain.rs:204-237) and the pair's
// 2 x u32 (summed chain length, number of chains: avg_chain_int_len's terms, chain.rs:244-249).
static void select_out(std::vector<ChainInterval>& good, uint64_t n_chunks, uint32_t c, uint32_t k, int switched,
                       int64_t* iv_out, uint32_t* hits, uint32_t* chunk_acc, uint32_t* pair_sums) {
  std::vector<uint8_t> kept;
  std::vector<uint32_t> h;
  auto per_chunk = get_nonoverlapping_chains(good, n_chunks, &kept, &h);
  for (size_t i = 0; i < good.size(); i++) {
    const ChainInterval& x = good[i];
    int64_t* o = iv_out + 11 * i;
    o[0] = (int64_t)x.score; o[1] = (int64_t)x.num_anchors; o[2] = x.q0; o[3] = x.q1; o[4] = x.r0; o[5] = x.r1;
    o[6] = (int64_t)x.ref_contig; o[7] = (int64_t)x.query_contig; o[8] = (int64_t)x.chunk_id; o[9] = x.reverse_chain;
    o[10] = kept[i];
    hits[2 * i] = h[2 * i]; hits[2 * i + 1] = h[2 * i + 1];
  }
  for (uint64_t ch = 0; ch < n_chunks; ch++) {
    const ChunkStats s = chunk_stats(per_chunk[ch], {}, c, k, MIN_LENGTH_COVER, switched != 0);
    const uint32_t row[5] = {(uint32_t)s.total_anchors, s.rq0, s.rq1, s.tbcq, s.n_int};
    memcpy(chunk_acc + 5 * ch, row, sizeof(row));
  }
  chain_len_sums(per_chunk, c, k, pair_sums, pair_sums + 1);
}

static MapParams unit_map_params(uint32_t c, uint32_t k) {
  Sketch unit;
  unit.c = c; unit.k = k;
  return map_params_from_sketch(unit, CommandParams(), -1);
}

// One pair's chunks: chunk i holds anchors chunk_off[i] .. chunk_off[i + 1] of a5 (5 x u32 per anchor: query_contig,
// query_pos, ref_contig, ref_pos, reverse), each chunk sorted as get_anchors leaves it.  Per anchor: score (i64) and
// chunk-local pointer; the sorted intervals go to iv_out / hits (capacity: n_anchors / 3 intervals), *n_iv = their number;
// the rest as select_out.
int orc_chain_chunks(uint32_t c, uint32_t k, int switched, uint64_t n_chunks, const uint64_t* chunk_off, const uint32_t* a5,
                     int64_t* score, uint32_t* pointer, int64_t* iv_out, uint32_t* hits, uint64_t* n_iv, uint32_t* chunk_acc,
                     uint32_t* pair_sums) {
  const MapParams mp = unit_map_params(c, k);
  std::vector<std::vector<Anchor>> chunks(n_chunks);
  for (uint64_t ch = 0; ch < n_chunks; ch++)
    for (uint64_t i = chunk_off[ch]; i < chunk_off[ch + 1]; i++) {
      const uint32_t* x = a5 + 5 * i;
      chunks[ch].push_back(Anchor{x[0], x[1], x[2], x[3], x[4] != 0});
    }
  std::vector<double> sc;
  std::vector<uint32_t> ptr;
  std::vector<ChainInterval> good = chain_chunks(chunks, mp, &sc, &ptr);
  for (size_t i = 0; i < sc.size(); i++) { score[i] = (int64_t)sc[i]; pointer[i] = ptr[i]; }
  *n_iv = good.size();
  select_out(good, n_chunks, c, k, switched, iv_out, hits, chunk_acc, pair_sums);
  return 0;
}

// The selection alone on n given intervals, 10 x i64 each (the orc_debug_intervals fields without `kept`), chunk ids below
// n_chunks; outputs as orc_chain_chunks (n intervals).
int orc_select_intervals(uint32_t c, uint32_t k, int switched, uint64_t n_chunks, uint64_t n, const int64_t* iv_in,
                         int64_t* iv_out, uint32_t* hits, uint32_t* chunk_acc, uint32_t* pair_sums) {
  std::vector<ChainInterval> good(n);
  for (uint64_t i = 0; i < n; i++) {
    const int64_t* x = iv_in + 10 * i;
    ChainInterval& v = good[i];
    v.score = (double)x[0]; v.num_anchors = (size_t)x[1];
    v.q0 = (uint32_t)x[2]; v.q1 = (uint32_t)x[3]; v.r0 = (uint32_t)x[4]; v.r1 = (uint32_t)x[5];
    v.ref_contig = (size_t)x[6]; v.query_contig = (size_t)x[7]; v.chunk_id = (size_t)x[8]; v.reverse_chain = x[9] != 0;
    v.overlap = 0;
  }
  select_out(good, n_chunks, c, k, switched, iv_out, hits, chunk_acc, pair_sums);
  return 0;
}

float orc_gbdt_predict(int model, const float* x) { return gbdt_predict(model, x); }

// final_estimate on a sorted (est, weight) list of n entries; quant_q / quant_r = {q10, q50, q90}; model -1 none, 0 C125,
// 1 C200.  The cutoffs and trim mode come from cmd as map_params_from_sketch takes them.
int orc_final_estimate(const double* est, const uint64_t* weight, uint64_t n, uint32_t total_query_bases,
                       uint32_t avg_chain_int_len, uint64_t query_total_len, uint64_t ref_total_len, const float* quant_q,
                       const float* quant_r, const orc_cmd* cmd, int model, orc_result* out) {
  std::vector<std::pair<double, size_t>> ests(n);
  for (uint64_t i = 0; i < n; i++) ests[i] = {est[i], (size_t)weight[i]};
  Sketch unit;
  unit.c = 125; unit.k = 15;
  MapParams mp = map_params_from_sketch(unit, to_cp(cmd), model);
  to_res(final_estimate(ests, total_query_bases, avg_chain_int_len, query_total_len, ref_total_len, quant_q, quant_r, mp),
         0, 0, out);
  return 0;
}

// chunk_estimate over n chunks of 8 x u32 each (total_anchors, rq0, rq1, tbcq, n_int, n_seeds, num_in, upper_lower), the form of
// sk_debug_chunk_estimate: est, weight and valid = 0 (no estimate), 1 (estimate) or 3 (estimate, filter applied)
int orc_chunk_estimate(uint64_t n, const uint32_t* in, uint32_t c, uint32_t k, double* est, uint32_t* weight, uint32_t* valid) {
  for (uint64_t i = 0; i < n; i++) {
    const uint32_t* x = in + 8 * i;
    ChunkStats s;
    s.total_anchors = x[0]; s.rq0 = x[1]; s.rq1 = x[2]; s.tbcq = x[3]; s.n_int = x[4];
    s.n_seeds = x[5]; s.num_in = x[6]; s.upper_lower = x[7];
    chunk_estimate(s, c, k, MIN_LENGTH_COVER);
    est[i] = s.est; weight[i] = (uint32_t)s.weight; valid[i] = s.valid ? (s.filtered ? 3u : 1u) : 0u;
  }
  return 0;
}

// ---- drivers ----------------------------------------------------------------------------------------
static int emit(const std::vector<PairResult>& v, orc_result** out, uint64_t* n) {
  orc_result* arr = (orc_result*)malloc(sizeof(orc_result) * (v.size() + 1));
  for (size_t i = 0; i < v.size(); i++) to_res(v[i].r, v[i].ref_id, v[i].query_id, &arr[i]);
  *out = arr; *n = v.size();
  return 0;
}
int orc_triangle(void** sk, int n, const orc_cmd* cmd, int threads, orc_result** out, uint64_t* n_out,
                 uint64_t* n_chained, double* t_screen, double* t_chain) {
  std::vector<const Sketch*> v;
  for (int i = 0; i < n; i++) v.push_back((Sketch*)sk[i]);
  return emit(triangle(v, to_cp(cmd), threads, n_chained, t_screen, t_chain), out, n_out);
}
int orc_dist(void** refs, int nr, void** queries, int nq, const orc_cmd* cmd, int use_index, int threads,
             orc_result** out, uint64_t* n_out) {
  std::vector<const Sketch*> r, q;
  for (int i = 0; i < nr; i++) r.push_back((Sketch*)refs[i]);
  for (int i = 0; i < nq; i++) q.push_back((Sketch*)queries[i]);
  return emit(dist(r, q, to_cp(cmd), use_index != 0, threads), out, n_out);
}
int orc_search(void** refs, int nr, void** queries, int nq, const orc_cmd* cmd, int use_index, int threads,
               orc_result** out, uint64_t* n_out) {
  std::vector<const Sketch*> r, q;
  for (int i = 0; i < nr; i++) r.push_back((Sketch*)refs[i]);
  for (int i = 0; i < nq; i++) q.push_back((Sketch*)queries[i]);
  return emit(search(r, q, to_cp(cmd), use_index != 0, threads), out, n_out);
}

}  // extern "C"

// seed ONE contig of any length with either semantics (no MIN_LENGTH_CONTIG rule; used for the reference's
// unit vectors tests/tests.rs:130-157 which call the seeders directly)
extern "C" void* orc_seed_one_contig(const uint8_t* s, uint64_t n, uint64_t c, uint64_t k, uint64_t marker_c, int avx2sem) {
  orc::SketchParams sp; sp.c = c; sp.k = k; sp.marker_c = marker_c;
  orc::Sketch* sk = new orc::Sketch();
  sk->c = c; sk->k = k; sk->marker_c = c;
  sk->contigs.push_back("contig0");
  sk->contig_lengths.push_back((uint32_t)n);
  sk->total_sequence_length = n;
  if (avx2sem) orc::fmh_seeds_avx2sem(s, n, sp, 0, *sk);
  else orc::fmh_seeds_scalar(s, n, sp, 0, *sk);
  return sk;
}

// sketch n_genomes genomes laid out like sk_sketch_batch's input, threads over genomes (the reference's own parallel
// structure, src/file_io.rs:149); handles are written to out[0..n_genomes)
extern "C" int orc_sketch_many(const uint8_t* bases, const uint64_t* contig_off, const uint32_t* genome_of_contig, uint32_t n_contigs,
                               uint32_t n_genomes, uint64_t c, uint64_t k, uint64_t marker_c, int threads, void** out) {
  orc::SketchParams sp; sp.c = c; sp.k = k; sp.marker_c = marker_c;
  std::vector<uint32_t> first(n_genomes + 1, n_contigs);
  for (uint32_t i = n_contigs; i-- > 0;) first[genome_of_contig[i]] = i;
  for (uint32_t g = n_genomes; g-- > 0;) if (first[g] == n_contigs && g + 1 <= n_genomes) first[g] = first[g + 1];
#pragma omp parallel for schedule(dynamic, 1) num_threads(threads > 0 ? threads : 1)
  for (long g = 0; g < (long)n_genomes; g++) {
    std::vector<std::pair<const uint8_t*, size_t>> ctgs;
    for (uint32_t i = first[g]; i < first[g + 1]; i++) ctgs.push_back({bases + contig_off[i], (size_t)(contig_off[i + 1] - contig_off[i])});
    char name[32];
    snprintf(name, sizeof(name), "g%06ld", g);
    out[g] = new orc::Sketch(orc::sketch_from_contigs(name, ctgs, nullptr, sp, true));
  }
  return 0;
}
