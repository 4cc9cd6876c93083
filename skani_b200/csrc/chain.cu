// chain.cu -- per-pair ANI estimation on the device: seed intersection -> anchors -> chunking -> banded chaining ->
// chain intervals -> greedy non-overlap selection -> per-chunk identities -> ANI / AF / std / bootstrap CI -> GBDT.
//
// Replaces chain::chain_seeds (reference src/chain.rs:144-171) with its callees get_anchors (:608-836),
// chain_anchors_ani (:838-896), get_chain_intervals (:939-1007), get_nonoverlapping_chains (:1008-1099),
// calculate_ani (:173-555), bootstrap_interval (:57-86) and regression::predict_from_ani_res (src/regression.rs:30-64).
//
// Data layout (HBM): both genomes of a pair are flat sorted arrays (sk_internal.h).  The query-role genome is
// streamed in (contig, pos) order and probed against the other genome's distinct k-mer array, so anchors come out
// already in the reference's sorted order (query_contig, query_pos, ref_contig, ref_pos, reverse) with no per-pair sort.
// Pairs are processed in batches; every stage is one kernel over the batch:
//   probe_kernel   (block/tile)  k-mer lookup per query record, multiplicity filters, anchor count per pair
//   chunk_anchor_kernel (block/pair) anchor offsets + 20 kb chunk assignment (segmented scans, closed form of the
//                  sequential loop) + anchors + chunk descriptors; chunk_compact_kernel packs the descriptors
//   dp_kernel      (thread/chunk) banded DP, chain components, chain intervals
//   select_kernel  (block/pair)  bitonic sort of intervals (descending derived order), greedy non-overlap filter
//   chunkstat_kernel (thread/chunk) seeds inside the padded interval union -> per-chunk identity
//   final_kernel   (block/pair)  sorted (est, weight) -> trimmed weighted mean, AF, std, bootstrap, cutoffs, GBDT
//   mapping_scan_kernel + mapping_emit_kernel (sk_chain_pairs_mappings only) kept intervals -> sorted sk_mapping records
#include <cub/cub.cuh>

#include <algorithm>
#include <cmath>
#include <cstdlib>
#include <cstring>
#include <limits>
#include <numeric>

#include "chain_core.cuh"
#include "mapping_core.cuh"
#include "sk_internal.h"

namespace sk {

namespace tables {
#include "gbdt_tables.inc"
}

__constant__ unsigned char c_gbdt_feat[2][1365];
__constant__ float c_gbdt_thr[2][1365];
__constant__ float c_gbdt_leaf[2][1560];
__constant__ float c_gbdt_shrink[2];
__constant__ float c_gbdt_bias[2];

struct SetView {
  const uint32_t *pv_kmer, *pv_pos, *pv_cc;
  const uint16_t* pv_mult;
  const uint32_t *kv_pos, *kv_cc, *ukmer, *ustart, *ctg_rec_off, *ubucket;
  const unsigned long long* htab;
};
struct GenomeMeta {
  uint64_t seed_off, uk_off, ctg_off;  // bases into the set arrays (ustart base = uk_off + g, ctg_rec_off base = ctg_off + g)
  uint32_t n_rec, n_uk, n_ctg, g;
  uint64_t total_len;
  uint32_t q10, q50, q90, pad;
  uint64_t ht_off;   // k-mer hash table of the genome (probe kernel); ht_cap == 0 => bucket search
  uint32_t ht_cap;
  uint32_t max_chunks;   // sum over contigs of ceil(len / FRAGMENT_LENGTH): no pair with this genome in the query role has more chunks
};
struct PairDesc {
  uint32_t qset, qg, rset, rg;  // query-role (iterated + chunked) and ref-role (probed) genome: set 0 = refs, 1 = queries
  uint32_t ref_idx, query_idx;
  uint32_t switched, valid;
  uint64_t rec_off;             // offset of this pair's slice in the per-record workspace
  uint64_t chunk_off;           // offset of this pair's slice in the chunk staging arrays
  uint32_t max_chunks, pad;     // bound on the pair's chunks = size of that slice (GenomeMeta::max_chunks of the query role)
};
struct ChainParams {
  uint32_t c, k, band, ushift;
  int32_t robust, median, model;  // model: -1 none, 0 C125, 1 C200
  double frac_cover_cutoff, both_frac_cover_cutoff;
};

// per-batch workspace (device pointers)
struct Workspace {
  // per record slot of the query-role genome (PairDesc::rec_off slices): probe tile j of a pair writes its hit records, in
  // record order, to slots [j * TILE, j * TILE + tile_hits[j]) of the pair's slice
  uint2* hit;             // .x = start of the matching group in the ref-role k-mer view, .y = record's index in its tile | nh << 10
  // per probe tile (tile_off indexing)
  uint32_t* tile_hits;    // hit records of the tile; chunk_anchor_kernel turns a pair's counts into pair-local exclusive offsets
  uint32_t* rec_cnt;      // TILE / 32 words per tile: bit i of word w = record 32 w + i is "counted" (enters seeds_in_chunk)
  // per pair
  uint32_t* tile_off;                    // exclusive prefix of the pairs' probe tiles (probe_kernel block -> pair), B + 1 entries
  uint32_t *pairA, *pairC;               // anchors, chunks
  uint64_t *pairAbase, *pairCbase, *pairIbase;  // exclusive prefix sums over the batch (anchors, chunks, interval capacity)
  uint32_t* pair_nint;
  uint32_t *pair_sumlen, *pair_nchains, *pair_tqb_ns;
  // per anchor
  AnchorRec* anc;
  int32_t* score;
  uint32_t *ptr, *depth;
  unsigned long long* rootkey;
  // per chunk, as chunk_anchor_kernel writes them: slices of PairDesc::max_chunks entries at PairDesc::chunk_off
  uint64_t* stg_first;
  uint32_t* stg_qctg;
  int64_t *stg_lo, *stg_hi;
  // per chunk
  uint64_t* chunk_first;   // batch-global anchor index (+ sentinel)
  uint32_t *chunk_pair, *chunk_qctg;
  uint32_t *chunk_size, *chunk_size_sorted, *chunk_id, *chunk_perm;   // DP load balance: chunks sorted by size
  int64_t *chunk_lo, *chunk_hi;  // seeds of the chunk: lo < pos <= hi
  uint32_t *acc_total, *acc_rq0, *acc_rq1, *acc_tbcq, *acc_nint, *chunk_head;
  double* chunk_est;
  uint32_t* chunk_w;
  uint8_t* chunk_valid;    // 0 no estimate, 1 estimate, 3 estimate after the putative-ANI filter
  uint32_t* chunk_nseeds;
  // per interval (capacity floor(A/3) per pair)
  IntervalKey* iv;
  uint32_t* iv_order;   // sorted order (indices local to the pair's slice)
  unsigned long long* iv_keys;  // primary sort keys for the global-memory sort fallback
  uint8_t* iv_kept;
  uint32_t* iv_next;
  uint32_t* acc_list;   // accepted interval indices (greedy)
  // per pair estimates scratch (sorted est/weight), capacity = chunks
  double* est_sorted;
  uint32_t* w_sorted;
};

constexpr int CT = 256;       // threads per block for block-per-pair kernels
constexpr int ITEMS = 4;

// ------------------------------------------------------------------------------------------------------------
// K1: probe
// ------------------------------------------------------------------------------------------------------------
// 1-D bulk copy (TMA, cp.async.bulk) global -> shared memory, completion signalled on an mbarrier: used to stage the whole
// k-mer table of a SMALL ref-role genome (<= 2048 entries = 16 KB: viruses, plasmids, single contigs -- BASELINE.json
// configs[4]) so that its probes hit shared memory instead of L2.  A/B switch SK_PROBE_TMA.
__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void bulk_load_to_smem(void* dst_smem, const void* src_gmem, uint32_t bytes, unsigned long long* bar) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
               ::"r"(smem_u32(dst_smem)), "l"(src_gmem), "r"(bytes), "r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ void mbar_wait(unsigned long long* bar, uint32_t parity) {
  asm volatile(
      "{\n"
      ".reg .pred p;\n"
      "WAIT_%=:\n"
      "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n"
      "@p bra DONE_%=;\n"
      "bra WAIT_%=;\n"
      "DONE_%=:\n"
      "}\n" ::"r"(smem_u32(bar)), "r"(parity) : "memory");
}
constexpr uint32_t PROBE_STAGE_ENTRIES = 2048;   // 16 KB: fits the (otherwise unused) bucket-index array of the block

constexpr uint32_t TILE = CT * ITEMS;            // query records per probe_kernel block / hit records per chunk_anchor_kernel step
static_assert(TILE / 32 == 32, "probe_kernel offsets a tile's 32 (item, warp) hit groups with one warp scan");
constexpr int PROBE_MINB = 4;                    // resident blocks per SM (register caps through __launch_bounds__)
constexpr int CHUNK_ANCHOR_MINB = 3;

// One block per TILE-record tile of the batch (PairDesc::rec_off slices, tile_off = tiles per pair): the tiles of a pair are
// independent, so nothing is carried between tiles.  The tile writes its hit records compacted in record order (warp ballots,
// per-warp counts in shared memory) with their count in tile_hits, and the "counted" bit of every record to rec_cnt (one
// ballot word per warp and item: 32 consecutive records).  The tile's anchor count goes to pairA with one atomic (integer
// sum: order-free).
// STAGED = the batch is dominated by small ref-role genomes: their tables are bulk-copied to shared memory (generic loads);
// otherwise every probe is a read-only global load.
template <bool STAGED, int MINB>
__global__ void __launch_bounds__(CT, MINB)
probe_kernel(const PairDesc* __restrict__ pairs, uint32_t n_pairs, SetView s0, SetView s1, const GenomeMeta* __restrict__ m0,
             const GenomeMeta* __restrict__ m1, ChainParams prm, Workspace ws) {
  __shared__ __align__(16) uint32_t s_bucket[UBUCKETS + 4];
  __shared__ __align__(8) unsigned long long s_bar;
  __shared__ uint32_t s_warp_sum[CT / 32];
  __shared__ uint32_t s_group_hits[ITEMS * CT / 32];
  // the tile's pair: the last p with tile_off[p] <= blockIdx.x (pairs without records own no tiles)
  uint32_t plo = 0, phi = n_pairs;
  while (phi - plo > 1) {
    const uint32_t mid = (plo + phi) >> 1;
    if (__ldg(ws.tile_off + mid) <= blockIdx.x) plo = mid; else phi = mid;
  }
  const uint32_t p = plo;
  const PairDesc pd = pairs[p];
  // the fields are selected one by one: a reference to s0 / s1 would copy both views to the stack of every thread
  const uint32_t* __restrict__ q_kmer = pd.qset ? s1.pv_kmer : s0.pv_kmer;
  const uint16_t* __restrict__ q_mult = pd.qset ? s1.pv_mult : s0.pv_mult;
  const GenomeMeta qm = (pd.qset ? m1 : m0)[pd.qg];
  const GenomeMeta rm = (pd.rset ? m1 : m0)[pd.rg];
  const uint32_t t0 = (blockIdx.x - __ldg(ws.tile_off + p)) * TILE;
  const uint32_t* __restrict__ ruk = (pd.rset ? s1.ukmer : s0.ukmer) + rm.uk_off;
  const uint32_t* __restrict__ rus = (pd.rset ? s1.ustart : s0.ustart) + rm.uk_off + rm.g;
  const uint32_t nuk = rm.n_uk;
  const bool use_hash = rm.ht_cap != 0;
  const unsigned long long* htab = (pd.rset ? s1.htab : s0.htab) + rm.ht_off;
  const uint32_t ht_mask = (rm.ht_cap >> 2) - 1;        // in 4-entry buckets
  if (STAGED && use_hash && rm.ht_cap <= PROBE_STAGE_ENTRIES) {   // block-uniform
    unsigned long long* s_tab = (unsigned long long*)s_bucket;
    if (threadIdx.x == 0) {
      asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(&s_bar)), "r"(1) : "memory");
      asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
      bulk_load_to_smem(s_tab, htab, rm.ht_cap * 8u, &s_bar);     // table offsets and sizes are multiples of 16 entries
    }
    __syncthreads();          // the barrier is initialised before anybody polls it
    mbar_wait(&s_bar, 0);
    htab = s_tab;
  }
  const uint32_t ht_shift = use_hash ? (32u - (uint32_t)__ffs((int)(rm.ht_cap >> 2)) + 1u) : 32u;   // 32 - log2(buckets); capacity >= 16 entries
  if (!use_hash) {  // fallback (genomes with >= 2^20 records): bucket index (16 KB) staged in shared memory
    // a genome without seed k-mers has neither a table nor a bucket index (the set may have none at all): every probe misses
    const uint32_t* gb = (pd.rset ? s1.ubucket : s0.ubucket) + (size_t)rm.g * (UBUCKETS + 1);
    for (uint32_t b = threadIdx.x; b <= UBUCKETS; b += CT) s_bucket[b] = nuk ? gb[b] : 0u;
    __syncthreads();
  }
  uint32_t hn[ITEMS], hr[ITEMS], hc[ITEMS];   // per record: anchors (nh), ref group start, counted
  // record t = t0 + it * CT + threadIdx.x: every load of the tile is coalesced
  if (use_hash) {
    // one 32-byte BUCKET (4 entries = one memory sector) per record: a probe almost never needs a second access, so the
    // lanes of a warp finish together (with one entry per step the warp waited for its longest probe chain).  The ITEMS probes of a thread are independent.
    uint32_t kmer[ITEMS], bidx[ITEMS];
    ulonglong2 ea[ITEMS], eb[ITEMS];
    bool live[ITEMS];
    const ulonglong2* __restrict__ tb2 = (const ulonglong2*)htab;
#pragma unroll
    for (int it = 0; it < ITEMS; it++) {
      const uint32_t t = t0 + it * CT + threadIdx.x;
      live[it] = false; kmer[it] = 0; bidx[it] = 0;
      ea[it] = make_ulonglong2(0ull, 0ull); eb[it] = ea[it];
      if (t < qm.n_rec) {
        kmer[it] = q_kmer[qm.seed_off + t];
        live[it] = q_mult[qm.seed_off + t] <= prm.band;   // query positions > band: dropped entirely (src/chain.rs:676-678)
        bidx[it] = (kmer[it] * 0x9E3779B1u) >> ht_shift;
      }
    }
#pragma unroll
    for (int it = 0; it < ITEMS; it++)
      if (live[it]) {
        if (STAGED) { ea[it] = tb2[2 * bidx[it]]; eb[it] = tb2[2 * bidx[it] + 1]; }
        else { ea[it] = __ldg(tb2 + 2 * bidx[it]); eb[it] = __ldg(tb2 + 2 * bidx[it] + 1); }
      }
#pragma unroll
    for (int it = 0; it < ITEMS; it++) {
      uint32_t nh = 0, rst = 0, counted = 0;
      if (live[it]) {
        unsigned long long e = 0ull;
        uint32_t b = bidx[it];
        ulonglong2 x = ea[it], y = eb[it];
        for (;;) {
          if ((uint32_t)(x.x >> 32) == kmer[it] && x.x != 0ull) { e = x.x; break; }
          if ((uint32_t)(x.y >> 32) == kmer[it] && x.y != 0ull) { e = x.y; break; }
          if ((uint32_t)(y.x >> 32) == kmer[it] && y.x != 0ull) { e = y.x; break; }
          if ((uint32_t)(y.y >> 32) == kmer[it] && y.y != 0ull) { e = y.y; break; }
          if (y.y == 0ull) break;                            // buckets fill front to back: an empty last slot ends the chain
          b = (b + 1) & ht_mask;                             // full bucket without the key: the key may have spilled over
          if (STAGED) { x = tb2[2 * b]; y = tb2[2 * b + 1]; } else { x = __ldg(tb2 + 2 * b); y = __ldg(tb2 + 2 * b + 1); }
        }
        if (e != 0ull) {
          const uint32_t cntr = (uint32_t)e & 0xFFFu;        // saturated at 4095 > any band
          if (cntr <= prm.band) { counted = 1; nh = cntr; rst = (uint32_t)(e >> 12) & 0xFFFFFu; }  // else dropped (:695-697)
        } else {
          counted = 1;                                       // no hit: position still counts (:684-687)
        }
      }
      hn[it] = nh; hr[it] = rst; hc[it] = counted;
    }
  } else {
    uint32_t kmer[ITEMS], lo[ITEMS], hi[ITEMS], bend[ITEMS];
    bool live[ITEMS];
    // the ITEMS searches of a thread advance in lock-step so that their (L2-latency) loads overlap
#pragma unroll
    for (int it = 0; it < ITEMS; it++) {
      const uint32_t t = t0 + it * CT + threadIdx.x;
      kmer[it] = 0; lo[it] = hi[it] = bend[it] = 0; live[it] = false;
      if (t < qm.n_rec) {
        kmer[it] = q_kmer[qm.seed_off + t];
        const uint32_t mq = q_mult[qm.seed_off + t];
        if (mq <= prm.band) {                          // query positions > band: dropped entirely (src/chain.rs:676-678)
          const uint32_t bk = kmer[it] >> prm.ushift;
          lo[it] = s_bucket[bk]; hi[it] = bend[it] = s_bucket[bk + 1];
          live[it] = true;
        }
      }
    }
    bool any = true;
    while (any) {
      any = false;
#pragma unroll
      for (int it = 0; it < ITEMS; it++) {
        if (live[it] && lo[it] < hi[it]) {
          const uint32_t mid = (lo[it] + hi[it]) >> 1;
          if (ruk[mid] < kmer[it]) lo[it] = mid + 1; else hi[it] = mid;
          any = true;
        }
      }
    }
#pragma unroll
    for (int it = 0; it < ITEMS; it++) {
      uint32_t nh = 0, rst = 0, counted = 0;
      if (live[it]) {
        if (lo[it] < bend[it] && lo[it] < nuk && ruk[lo[it]] == kmer[it]) {
          const uint32_t s = rus[lo[it]], cntr = rus[lo[it] + 1] - s;
          if (cntr <= prm.band) { counted = 1; nh = cntr; rst = s; }  // else dropped entirely (:695-697)
        } else {
          counted = 1;                                 // no hit: position still counts (:684-687)
        }
      }
      hn[it] = nh; hr[it] = rst; hc[it] = counted;
    }
  }
  // The lanes of warp w for item it hold the 32 consecutive records it * CT + 32 w + lane of the tile: one ballot word
  // each for rec_cnt and for the hit mask.  Group (it, w) precedes group (it', w') in record order iff it * 8 + w is smaller.
  const unsigned FULL = 0xFFFFFFFFu;
  const uint32_t lane = threadIdx.x & 31u, w = threadIdx.x >> 5;
  uint32_t hm[ITEMS], sum = 0;
#pragma unroll
  for (int it = 0; it < ITEMS; it++) {
    hm[it] = __ballot_sync(FULL, hn[it] != 0);
    const uint32_t cm = __ballot_sync(FULL, hc[it] != 0);
    if (lane == 0) {
      ws.rec_cnt[(size_t)blockIdx.x * (TILE / 32) + it * (CT / 32) + w] = cm;
      s_group_hits[it * (CT / 32) + w] = __popc(hm[it]);
    }
    sum += hn[it];
  }
  sum = __reduce_add_sync(FULL, sum);
  if (lane == 0) s_warp_sum[w] = sum;
  __syncthreads();
  // every warp scans the 32 group counts itself: exclusive offset of each group among the tile's hits
  const uint32_t gv = s_group_hits[lane];
  uint32_t ginc = gv;
#pragma unroll
  for (uint32_t o = 1; o < 32; o <<= 1) {
    const uint32_t x = __shfl_up_sync(FULL, ginc, o);
    if (lane >= o) ginc += x;
  }
  uint2* __restrict__ hv = ws.hit + pd.rec_off + t0;
  const uint32_t lt = (1u << lane) - 1u;
#pragma unroll
  for (int it = 0; it < ITEMS; it++) {
    const uint32_t gbase = __shfl_sync(FULL, ginc - gv, it * (CT / 32) + w);
    if (hn[it]) hv[gbase + __popc(hm[it] & lt)] = make_uint2(hr[it], (it * CT + threadIdx.x) | (hn[it] << 10));
  }
  const uint32_t tile_total = __shfl_sync(FULL, ginc, 31);
  if (threadIdx.x == 0) {
    ws.tile_hits[blockIdx.x] = tile_total;
    uint32_t total = 0;
#pragma unroll
    for (int w = 0; w < CT / 32; w++) total += s_warp_sum[w];
    if (total) atomicAdd(&ws.pairA[p], total);
  }
}

// ------------------------------------------------------------------------------------------------------------
// K2: chunk assignment + anchors + chunk descriptors, block per pair, streaming the query-role genome's hit records (the
// probe's compacted per-tile lists) in steps of TILE hits.  Records without hits enter every scan as its identity, so only
// hit records are scanned.  Per hit record, with in-step block scans carried across steps: the pair-local offset of its first anchor (sum of nh),
// P0 / A0 of its contig (position / anchor offset of the contig's first hit, segmented "first" scan), need, and the
// contig-local chunk of its first and last anchor (segmented prefix min, the closed form in chain_core.cuh); then the
// chunk-start flags and chunk ids (sum).  Descriptors go to the pair's staging slice; chunk_compact_kernel packs them.
//
// Few memory round trips lie in series inside a step: the hits of step i + 1 are staged in shared memory (cp.async) while
// step i scans and emits, and the step's anchors are emitted anchor-parallel, one thread per anchor, so that the
// gathers of a round are independent of each other and of the round's stores.  What remains is mostly the instruction
// work of the four block scans (hence the branch-free FirstOp / MinOp).
// ------------------------------------------------------------------------------------------------------------
// 4-byte asynchronous copy global -> shared memory.  A thread waits for its own copies (wait_group); a barrier then
// publishes them to the block.
__device__ __forceinline__ void cp_async4(void* dst_smem, const void* src_gmem) {
  asm volatile("cp.async.ca.shared.global [%0], [%1], 4;" ::"r"(smem_u32(dst_smem)), "l"(src_gmem) : "memory");
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;" ::: "memory"); }
__device__ __forceinline__ void cp_async_wait_all_but_newest() { asm volatile("cp.async.wait_group 1;" ::: "memory"); }

static_assert(TILE == 1024, "ChunkAnchorSmem::arec and Workspace::hit pack an index in the step / tile into 10 bits");
struct __align__(16) RecTile {       // one step of hit records of the query-role genome
  uint32_t pos[TILE], cc[TILE];      // not copied for the padding slots after the pair's last hit
  uint32_t rs[TILE];
  uint32_t nh[TILE];                 // 0 for the padding slots
};
struct ChunkAnchorSmem {
  RecTile tile[2];                   // double buffer: step i + 1 is in flight while step i scans and emits
  // per hit record of the current step (index in the step), read by the threads that emit its anchors
  uint32_t clf[TILE];                // contig-local chunk of the record's first anchor
  uint32_t need[TILE];               // need | (the first anchor starts a chunk) << 31
  uint32_t cid[TILE];                // pair-local chunk id of the first anchor
  uint32_t p0[TILE];                 // P0 of the record's contig
  uint32_t arec[TILE];               // anchor of the current round -> its record | its index in the record << 10
};

// Stage the pair's hits [h0, min(h0 + TILE, H)) into b.  Hit h lies in probe tile j, the last tile with hoff[j] <= h (a
// tile without hits shares its offset with the next tile, so the search passes over it); its entry is read at once, and
// its record's pos / cc are copied asynchronously (increasing addresses inside the tile's window of TILE records).
// hoff: the pair's n_t tile offsets, written by this block (plain loads, not the read-only path).
__device__ __forceinline__ void stage_hit_step(RecTile& b, uint32_t h0, uint32_t H, const uint32_t* hoff, uint32_t n_t,
                                               const uint2* hv, const uint32_t* qpv, const uint32_t* qcv) {
  uint32_t h[ITEMS], j[ITEMS];
#pragma unroll
  for (int it = 0; it < ITEMS; it++) { h[it] = h0 + it * CT + threadIdx.x; j[it] = 0; }
  for (uint32_t len = n_t; len > 1;) {             // the ITEMS searches in lock-step: their loads overlap
    const uint32_t half = len >> 1;
#pragma unroll
    for (int it = 0; it < ITEMS; it++)
      if (hoff[j[it] + half] <= h[it]) j[it] += half;
    len -= half;
  }
#pragma unroll
  for (int it = 0; it < ITEMS; it++) {
    const uint32_t i = it * CT + threadIdx.x;
    uint32_t nh = 0;
    if (h[it] < H) {
      const uint32_t r0 = j[it] * TILE;                // the tile's first record = its first hit slot
      const uint2 e = hv[r0 + (h[it] - hoff[j[it]])];
      const uint32_t r = r0 + (e.y & (TILE - 1));
      cp_async4(&b.pos[i], qpv + r);
      cp_async4(&b.cc[i], qcv + r);
      b.rs[i] = e.x;
      nh = e.y >> 10;
    }
    b.nh[i] = nh;
  }
}

template <int MINB>
__global__ void __launch_bounds__(CT, MINB)
chunk_anchor_kernel(const PairDesc* __restrict__ pairs, SetView s0, SetView s1, const GenomeMeta* __restrict__ m0,
                    const GenomeMeta* __restrict__ m1, Workspace ws) {
  using ScanU = cub::BlockScan<uint32_t, CT, cub::BLOCK_SCAN_WARP_SCANS>;
  using ScanF = cub::BlockScan<FirstState, CT, cub::BLOCK_SCAN_WARP_SCANS>;
  using ScanM = cub::BlockScan<MinState, CT, cub::BLOCK_SCAN_WARP_SCANS>;
  // one storage per scan of a step: between two uses of a storage lie other block scans, whose barriers order the accesses
  __shared__ typename ScanU::TempStorage tmp_a, tmp_c;
  __shared__ typename ScanF::TempStorage tmp_f;
  __shared__ typename ScanM::TempStorage tmp_m;
  extern __shared__ __align__(16) unsigned char smem_raw[];
  ChunkAnchorSmem& S = *reinterpret_cast<ChunkAnchorSmem*>(smem_raw);
  const uint32_t p = blockIdx.x;
  const PairDesc pd = pairs[p];
  const uint32_t A_total = ws.pairA[p];
  if (!pd.valid || A_total == 0) {
    if (threadIdx.x == 0) ws.pairC[p] = 0;
    return;
  }
  const GenomeMeta qm = (pd.qset ? m1 : m0)[pd.qg];
  const GenomeMeta rm = (pd.rset ? m1 : m0)[pd.rg];
  const uint2* __restrict__ hv = ws.hit + pd.rec_off;
  // the fields are selected one by one (see probe_kernel)
  const uint32_t* __restrict__ qpv = (pd.qset ? s1.pv_pos : s0.pv_pos) + qm.seed_off;
  const uint32_t* __restrict__ qcv = (pd.qset ? s1.pv_cc : s0.pv_cc) + qm.seed_off;
  const uint32_t* __restrict__ rpv = (pd.rset ? s1.kv_pos : s0.kv_pos) + rm.seed_off;
  const uint32_t* __restrict__ rcv = (pd.rset ? s1.kv_cc : s0.kv_cc) + rm.seed_off;
  const uint64_t abase = ws.pairAbase[p], sbase = pd.chunk_off;
  AnchorRec* __restrict__ anc = ws.anc + abase;
  const uint32_t cmax = pd.max_chunks;
  // the probe's per-tile hit counts -> pair-local exclusive offsets (in place), H = the pair's hit records
  const uint32_t tb = ws.tile_off[p], n_t = ws.tile_off[p + 1] - tb;
  uint32_t* hoff = ws.tile_hits + tb;
  uint32_t H = 0;
  for (uint32_t j0 = 0; j0 < n_t; j0 += TILE) {
    uint32_t x[ITEMS], ex[ITEMS], agg;
#pragma unroll
    for (int it = 0; it < ITEMS; it++) {
      const uint32_t j = j0 + threadIdx.x * ITEMS + it;
      x[it] = j < n_t ? hoff[j] : 0u;
    }
    ScanU(tmp_a).ExclusiveSum(x, ex, agg);
#pragma unroll
    for (int it = 0; it < ITEMS; it++) {
      const uint32_t j = j0 + threadIdx.x * ITEMS + it;
      if (j < n_t) hoff[j] = H + ex[it];
    }
    H += agg;
    __syncthreads();                                // tmp_a is reused; the offsets are visible to the whole block
  }
  FirstState carryF; carryF.valid = 0; carryF.ctg = 0; carryF.p0 = 0; carryF.a0 = 0;
  MinState carryM; carryM.valid = 0; carryM.ctg = 0; carryM.v = 0;
  MinState identM; identM.valid = 0; identM.ctg = 0; identM.v = 0;
  uint32_t carryA = 0, carryC = 0;                  // anchors / chunk starts so far
  __shared__ uint32_t s_last_q, s_last_c;          // the pair's last hit record: its position, the chunk of its last anchor
  stage_hit_step(S.tile[0], 0, H, hoff, n_t, hv, qpv, qcv);
  cp_async_commit();
  uint32_t buf = 0;
  for (uint32_t h0 = 0; h0 < H; h0 += TILE, buf ^= 1u) {
    // the other buffer was last read before the previous step's final barrier
    if (h0 + TILE < H) stage_hit_step(S.tile[buf ^ 1u], h0 + TILE, H, hoff, n_t, hv, qpv, qcv);
    cp_async_commit();                              // possibly empty: the group before it is always this step's
    cp_async_wait_all_but_newest();
    __syncthreads();
    const RecTile& T = S.tile[buf];
    uint32_t nh[ITEMS], pos[ITEMS], cc[ITEMS];
    {
      const uint4 p4 = *reinterpret_cast<const uint4*>(&T.pos[threadIdx.x * ITEMS]);
      const uint4 c4 = *reinterpret_cast<const uint4*>(&T.cc[threadIdx.x * ITEMS]);
      const uint4 n4 = *reinterpret_cast<const uint4*>(&T.nh[threadIdx.x * ITEMS]);
      pos[0] = p4.x; pos[1] = p4.y; pos[2] = p4.z; pos[3] = p4.w;
      cc[0] = c4.x; cc[1] = c4.y; cc[2] = c4.z; cc[3] = c4.w;
      nh[0] = n4.x; nh[1] = n4.y; nh[2] = n4.z; nh[3] = n4.w;
#pragma unroll
      for (int it = 0; it < ITEMS; it++)
        if (!nh[it]) pos[it] = cc[it] = 0;          // padding slots: never copied
    }
    uint32_t aoff[ITEMS], aggA;
    ScanU(tmp_a).ExclusiveSum(nh, aoff, aggA);
    FirstState fs[ITEMS];
#pragma unroll
    for (int it = 0; it < ITEMS; it++) {
      aoff[it] += carryA;                           // pair-local offset of the record's first anchor
      fs[it].valid = nh[it] ? 1u : 0u; fs[it].ctg = cc[it] >> 1; fs[it].p0 = pos[it]; fs[it].a0 = aoff[it];
    }
    FirstState aggF;
    ScanF(tmp_f).InclusiveScan(fs, fs, FirstOp(), aggF);
    MinState ms[ITEMS];
    uint32_t need[ITEMS], al[ITEMS];
#pragma unroll
    for (int it = 0; it < ITEMS; it++) {
      ms[it] = identM;
      need[it] = al[it] = 0;
      if (nh[it]) {
        fs[it] = FirstOp()(carryF, fs[it]);
        need[it] = chunk_need(pos[it], fs[it].p0);
        al[it] = aoff[it] - fs[it].a0;             // contig-local index of the record's first anchor
        ms[it].valid = 1; ms[it].ctg = cc[it] >> 1;
        ms[it].v = record_min_key(need[it], al[it], nh[it]);
      }
    }
    carryF = FirstOp()(carryF, aggF);
    MinState exm[ITEMS], aggM;
    ScanM(tmp_m).ExclusiveScan(ms, exm, identM, MinOp(), aggM);
    uint32_t clf[ITEMS], cll[ITEMS], st[ITEMS], inc[ITEMS];
#pragma unroll
    for (int it = 0; it < ITEMS; it++) {
      clf[it] = cll[it] = st[it] = inc[it] = 0;
      if (nh[it]) {
        const MinState e = MinOp()(carryM, exm[it]);     // everything before this record
        const bool has_prev = e.valid && e.ctg == (cc[it] >> 1);
        clf[it] = chunk_local_of(al[it], has_prev, e.v, need[it]);
        cll[it] = chunk_local_of((uint64_t)al[it] + nh[it] - 1, has_prev, e.v, need[it]);
        st[it] = record_starts_chunk(al[it], has_prev, e.v, clf[it]);
        inc[it] = record_chunk_starts(st[it], clf[it], cll[it]);
      }
    }
    carryM = MinOp()(carryM, aggM);
    uint32_t exc[ITEMS], aggC;
    ScanU(tmp_c).ExclusiveSum(inc, exc, aggC);
#pragma unroll
    for (int it = 0; it < ITEMS; it++) {
      if (!nh[it]) continue;
      const uint32_t r = threadIdx.x * ITEMS + it;
      const uint32_t cid = carryC + exc[it] + st[it] - 1;   // chunk id of the record's first anchor
      S.clf[r] = clf[it];
      S.need[r] = need[it] | (st[it] << 31);                 // need < 2^18: positions are 32-bit
      S.cid[r] = cid;
      S.p0[r] = fs[it].p0;
      if (aoff[it] + nh[it] == A_total) { s_last_q = pos[it]; s_last_c = cid + (cll[it] - clf[it]); }
    }
    // The tile's anchors are the pair-local range [carryA, carryA + aggA), emitted in rounds of TILE: the records first
    // mark which of the round's anchors are theirs, then thread k * CT + threadIdx.x of the round emits anchor k * CT +
    // threadIdx.x (consecutive threads write consecutive anchors).  A record's anchors may span rounds.
    for (uint32_t base = 0; base < aggA; base += TILE) {
#pragma unroll
      for (int it = 0; it < ITEMS; it++) {
        if (!nh[it]) continue;
        const uint32_t lo = aoff[it] - carryA, r = threadIdx.x * ITEMS + it;
        const uint32_t j1 = min(lo + nh[it], base + TILE);
        for (uint32_t j = max(lo, base); j < j1; j++) S.arec[j - base] = r | ((j - lo) << 10);
      }
      __syncthreads();
      uint32_t ar[ITEMS], rpos[ITEMS], rcc[ITEMS];
#pragma unroll
      for (int k = 0; k < ITEMS; k++) {             // every gather of the round before any of its stores
        const uint32_t j = base + k * CT + threadIdx.x;
        ar[k] = rpos[k] = rcc[k] = 0;
        if (j < aggA) {
          ar[k] = S.arec[j - base];
          const uint32_t g = T.rs[ar[k] & (TILE - 1)] + (ar[k] >> 10);
          rpos[k] = __ldg(rpv + g);
          rcc[k] = __ldg(rcv + g);
        }
      }
#pragma unroll
      for (int k = 0; k < ITEMS; k++) {
        const uint32_t j = base + k * CT + threadIdx.x;
        if (j >= aggA) continue;
        const uint32_t r = ar[k] & (TILE - 1), u = ar[k] >> 10;
        const uint32_t qcc = T.cc[r], clf0 = S.clf[r], nd = S.need[r], rneed = nd & 0x7FFFFFFFu;
        AnchorRec a;
        a.qpos = T.pos[r]; a.rpos = rpos[k];
        a.rc = (rcc[k] & ~1u) | ((rcc[k] ^ qcc) & 1u);          // reverse_match = canonical differs (src/chain.rs:709)
        anc[carryA + j] = a;
        const uint32_t cl = anchor_chunk_local(clf0, u, rneed);
        const bool start = anchor_starts_chunk(clf0, u, rneed, (nd >> 31) != 0);
        const uint32_t mycid = S.cid[r] + (cl - clf0);
        if (start && mycid < cmax) {                             // chunk start: write its descriptor
          const uint64_t c = sbase + mycid;
          const uint32_t p0 = S.p0[r];
          ws.stg_first[c] = abase + carryA + j;
          ws.stg_qctg[c] = qcc >> 1;
          ws.stg_lo[c] = chunk_window_lo(p0, cl);
          ws.stg_hi[c] = chunk_window_hi(p0, cl);
        }
      }
      __syncthreads();                              // arec, the per-record arrays and this tile buffer are reused
    }
    carryA += aggA;
    carryC += aggC;
  }
  // the pair's last chunk is never closed by the loop: it keeps seeds up to its last anchor (src/chain.rs:796-824).
  // Patched after every descriptor of this pair has been written, whichever threads wrote them (same block; A_total > 0,
  // so exactly one record set s_last_q / s_last_c).
  __syncthreads();
  if (threadIdx.x == 0) {
    if (s_last_c < cmax) ws.stg_hi[sbase + s_last_c] = (int64_t)s_last_q;
    ws.pairC[p] = carryC;                         // > max_chunks: run_batch reports the error, nothing was written out of range
  }
}

// ------------------------------------------------------------------------------------------------------------
// K2b: chunk descriptors from the staging slices into the dense batch arrays the later kernels read, block per pair
// ------------------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(CT)
chunk_compact_kernel(const PairDesc* __restrict__ pairs, Workspace ws) {
  const uint32_t p = blockIdx.x;
  const uint32_t n = ws.pairC[p];
  const uint64_t src = pairs[p].chunk_off, dst = ws.pairCbase[p];
  for (uint32_t i = threadIdx.x; i < n; i += CT) {
    ws.chunk_first[dst + i] = ws.stg_first[src + i];
    ws.chunk_pair[dst + i] = p;
    ws.chunk_qctg[dst + i] = ws.stg_qctg[src + i];
    ws.chunk_lo[dst + i] = ws.stg_lo[src + i];
    ws.chunk_hi[dst + i] = ws.stg_hi[src + i];
  }
}

// ------------------------------------------------------------------------------------------------------------
// K4: banded DP + chain extraction, one WARP per chunk, anchors and DP state held in registers.
//
// Lane l owns the anchors whose chunk index is congruent to l mod 32: register set s holds the anchor of block
// (current block - s).  For the anchor i = 32 b + m being scored, every lane tests its own candidates j = 32 (b - s) + l
// (the reference's predecessor window j in [i - band, i), same ref contig, query gap <= 2500, src/chain.rs:853-880) against
// the anchor's fields broadcast from lane m; two REDUX reductions pick the maximal score and, among those, the largest j
// (the reference's strict `>` scanning j downward).  Chain components are tracked with the closed form of the union-find
// (root / depth propagate through the winning predecessor); per-root statistics live in global memory at the root's slot.
// ------------------------------------------------------------------------------------------------------------
template <int NB, bool TAPS>
__global__ void __launch_bounds__(32)
dp_warp_kernel(uint64_t n_chunks, ChainParams prm, Workspace ws) {
  const unsigned FULL = 0xFFFFFFFFu;
  const uint32_t lane = threadIdx.x;
  const uint64_t c = blockIdx.x;
  if (c >= n_chunks) return;
  const uint64_t a0 = ws.chunk_first[c];
  const uint32_t n = (uint32_t)(ws.chunk_first[c + 1] - a0);
  const AnchorRec* __restrict__ a = ws.anc + a0;
  // per-root "best chain end" key = score << 32 | index, maintained with atomicMax: the maximum is the largest index
  // among the maximal scores, exactly the reference's pick (SURVEY App. A.8).  depth = anchors on the path to the root.
  unsigned long long* __restrict__ g_key = ws.rootkey + a0;
  uint32_t* __restrict__ g_depth = ws.depth + a0;
  const uint32_t band = prm.band;
  uint32_t q[NB], r[NB], rc[NB], rt[NB], dpth[NB];
  int32_t sc[NB];
  uint32_t my_ptr = 0;
#pragma unroll
  for (int s = 0; s < NB; s++) { q[s] = r[s] = rc[s] = rt[s] = dpth[s] = 0; sc[s] = 0; }
  for (uint32_t b0 = 0; b0 < n; b0 += 32) {
#pragma unroll
    for (int s = NB - 1; s > 0; s--) { q[s] = q[s - 1]; r[s] = r[s - 1]; rc[s] = rc[s - 1]; rt[s] = rt[s - 1]; dpth[s] = dpth[s - 1]; sc[s] = sc[s - 1]; }
    const uint32_t idx = b0 + lane;
    {
      AnchorRec x; x.qpos = 0; x.rpos = 0; x.rc = 0;
      if (idx < n) { x = a[idx]; g_key[idx] = (unsigned long long)idx; }   // every anchor starts as its own root, score 0
      q[0] = x.qpos; r[0] = x.rpos; rc[0] = x.rc; sc[0] = 0; rt[0] = idx; dpth[0] = 1;
      my_ptr = idx;
    }
    __syncwarp();
    const uint32_t mend = min(32u, n - b0);
    for (uint32_t m = 0; m < mend; m++) {
      const uint32_t i = b0 + m;
      AnchorRec cur;
      cur.qpos = __shfl_sync(FULL, q[0], m);
      cur.rpos = __shfl_sync(FULL, r[0], m);
      cur.rc = __shfl_sync(FULL, rc[0], m);
      int32_t best_ns = 0;
      uint32_t best_j1 = 0;  // j + 1 of this lane's best candidate
      // Exactly one of two adjacent register sets can hold a predecessor of i in this lane: set t when lane < m
      // (j = 32 (b - t) + lane < i in the same residue class), set t + 1 otherwise.  32-bit arithmetic throughout:
      // contig lengths are < 2^32 - 65536 (enforced at sketch time), so the unsigned range tests below are exact.
      const bool lo_set = lane < m;
#pragma unroll
      for (int t = 0; t < NB - 1; t++) {   // ascending t = descending j inside a lane: strict > keeps the largest j
        const uint32_t qs = lo_set ? q[t] : q[t + 1];
        const uint32_t rs = lo_set ? r[t] : r[t + 1];
        const uint32_t rcs = lo_set ? rc[t] : rc[t + 1];
        const int32_t scs = lo_set ? sc[t] : sc[t + 1];
        const uint32_t d = m + 32u * (uint32_t)t + (lo_set ? 0u : 32u) - lane;   // i - j >= 1
        const uint32_t j = i - d;                                               // wraps when the set is not filled yet
        const uint32_t dq = cur.qpos - qs;                                      // >= 0 inside a chunk (sorted)
        const uint32_t tr = cur.rpos - rs;
        const uint32_t dr = (cur.rc & 1u) ? (0u - tr) : tr;                     // src/chain.rs:580-584
        const uint32_t g = dr - dq;
        const bool ok = (d <= band) & (d <= i) &                                // window (:859-863) and j >= 0
                        (rcs == cur.rc) &                                       // same ref contig (:856) and same strand (:564)
                        (dq - 1u < BP_CHAIN_BAND) &                             // query_pos differs (:567) and dq <= 2500 (:859)
                        (dr - 1u < (uint32_t)MAX_LIN) &                         // 0 < dr <= 5000 (:586-592), ref_pos differs (:567)
                        (g + (uint32_t)MAX_GAP <= 2u * (uint32_t)MAX_GAP);      // |dr - dq| <= 300 (:594-597)
        const int32_t gi = (int32_t)g;
        const int32_t ns = scs + ANCHOR_SCORE - (gi < 0 ? -gi : gi);
        if (ok && ns > best_ns) { best_ns = ns; best_j1 = j + 1; }
      }
      const int32_t smax = __reduce_max_sync(FULL, best_ns);
      if (smax > 0) {   // uniform branch
        const uint32_t jw = __reduce_max_sync(FULL, (best_ns == smax) ? best_j1 : 0u) - 1;
        const int sidx = (int)(b0 >> 5) - (int)(jw >> 5);
        uint32_t rsel = rt[0], dsel = dpth[0];
#pragma unroll
        for (int s = 1; s < NB; s++) if (sidx == s) { rsel = rt[s]; dsel = dpth[s]; }
        const uint32_t root_i = __shfl_sync(FULL, rsel, jw & 31u);
        const uint32_t depth_i = __shfl_sync(FULL, dsel, jw & 31u) + 1;
        if (lane == m) { sc[0] = smax; rt[0] = root_i; dpth[0] = depth_i; my_ptr = jw; }
      }
    }
    // block epilogue: coalesced depth store; chained anchors push their (score, index) to their root
    if (idx < n) {
      g_depth[idx] = dpth[0];
      if (rt[0] != idx) atomicMax(&g_key[rt[0]], ((unsigned long long)(uint32_t)sc[0] << 32) | idx);
      if (TAPS) { ws.score[a0 + idx] = sc[0]; ws.ptr[a0 + idx] = my_ptr; }
    }
  }
  __threadfence_block();
  __syncwarp();
  // emit one interval per surviving chain (src/chain.rs:954-1005).  The len_of_set >= 3 test (:954-957) is implied by
  // num_anchors >= 3 (:974): a component has at least as many members as its best path.
  const uint32_t p = ws.chunk_pair[c];
  const uint32_t qctg = ws.chunk_qctg[c];
  const uint32_t chunk_local_id = (uint32_t)(c - ws.pairCbase[p]);
  for (uint32_t i = lane; i < n; i += 32) {
    if (((volatile uint32_t*)g_depth)[i] != 1) continue;            // not a root
    const unsigned long long key = ((volatile unsigned long long*)g_key)[i];
    const uint32_t b = (uint32_t)key, score = (uint32_t)(key >> 32);
    if (b == i) continue;                                            // singleton
    const uint32_t num_anchors = ((volatile uint32_t*)g_depth)[b];
    if (num_anchors < MIN_ANCHORS || (int32_t)score < MIN_SCORE) continue;
    const AnchorRec f = a[i], l = a[b];
    uint32_t r0 = f.rpos < l.rpos ? f.rpos : l.rpos, r1 = f.rpos < l.rpos ? l.rpos : f.rpos;
    IntervalKey key5 = make_interval((int32_t)score, num_anchors, f.qpos, l.qpos, r0, r1, f.rc >> 1, qctg, chunk_local_id, f.rc & 1u);
    uint32_t slot = atomicAdd(&ws.pair_nint[p], 1u);
    ws.iv[ws.pairIbase[p] + slot] = key5;
  }
}

// ------------------------------------------------------------------------------------------------------------
// K4b: the same DP with FOUR chunks per warp (8 lanes each), used when the band fits 3 candidates per lane (band <= 24,
// i.e. c >= 105).  With band = 20 a full warp per chunk leaves 12 lanes idle and spends most of its issue slots on the
// per-step bookkeeping; 8-lane groups evaluate 3 candidates per lane and amortise the bookkeeping over 4 anchors.
// Lane gl of a group owns the anchors congruent to gl mod 8; register set s holds the anchor of block (current - s).
// Group-wide arg-max = two 3-step xor-butterflies (max score, then largest j among the maxima).
//
// Chain bookkeeping.  A chunk of at most DP_SMEM_ANCHORS anchors keeps it in its group's slab of shared memory: one word per
// anchor, score << 16 | index << 8 | (depth - 1), which starts as the anchor's own (0, index, 0) and, at a root, ends as the
// shared-memory atomicMax over the root's chained anchors -- the maximum is the largest index among the maximal scores, and
// carries that end's depth.  A word whose index field is its own anchor is a singleton or not a root: no interval.  Longer
// chunks keep the per-anchor rootkey / depth arrays in global memory.  Field widths: index and depth - 1 < 256, score <=
// ANCHOR_SCORE * DP_SMEM_ANCHORS < 2^16.  224 covers every chunk of a `north` step (at most 215 anchors, DESIGN §3), and its
// 7 KB slab per warp (8 groups) still lets the 28 warps per SM that 72 registers allow be resident (28 x (7 + 1 reserved) KB).
// ------------------------------------------------------------------------------------------------------------
constexpr uint32_t DP_SMEM_ANCHORS = 224;
static_assert(DP_SMEM_ANCHORS <= 256 && (uint64_t)ANCHOR_SCORE * DP_SMEM_ANCHORS < (1u << 16), "dp_group_kernel's packed chain word");

template <bool TAPS, int GL, int NE, bool FULLBAND, int MINB>
__global__ void __launch_bounds__(32, MINB)
dp_group_kernel(uint64_t n_chunks, ChainParams prm, Workspace ws) {
  // FULLBAND: band == GL * NE, so every candidate distance the register sets can express is inside the band (no test needed)
  // GL lanes per chunk (8 or 4), 32 / GL chunks per warp.  Lane gl of a group owns the anchors congruent to gl mod GL;
  // register set s holds the anchor of block (current - s); a lane evaluates NE candidates per step, which covers every
  // predecessor distance d <= GL * NE (band = 20 at c = 125: NE = 5 with 4 lanes, 3 with 8).
  constexpr int NB = NE + 1;
  constexpr int LG = (GL == 8) ? 3 : 2;       // log2(GL)
  constexpr uint32_t GW = 32 / GL;            // chunks per warp
  const unsigned FULL = 0xFFFFFFFFu;
  const uint32_t lane = threadIdx.x, gl = lane & (GL - 1), gbase = lane & ~(uint32_t)(GL - 1);
  const uint64_t slot = (uint64_t)blockIdx.x * GW + (lane >> LG);
  const bool live = slot < n_chunks;
  const uint64_t c = live ? (uint64_t)ws.chunk_perm[slot] : 0;   // chunks sorted by size: the chunks of a warp are alike
  uint64_t a0 = 0;
  uint32_t n = 0;
  if (live) { a0 = ws.chunk_first[c]; n = (uint32_t)(ws.chunk_first[c + 1] - a0); }
  const AnchorRec* __restrict__ a = ws.anc + a0;
  unsigned long long* __restrict__ g_key = ws.rootkey + a0;
  uint32_t* __restrict__ g_depth = ws.depth + a0;
  __shared__ uint32_t s_chain[GW][DP_SMEM_ANCHORS];
  uint32_t* const s_word = s_chain[lane >> LG];
  const bool onchip = n <= DP_SMEM_ANCHORS;
  const uint32_t band = prm.band;
  // longest chunk of the warp bounds the common loop
  uint32_t nmax = n;
#pragma unroll
  for (int o = 16; o >= GL; o >>= 1) nmax = max(nmax, __shfl_xor_sync(FULL, nmax, o));
  uint32_t q[NB], r[NB], rc[NB], rt[NB], dpth[NB];
  int32_t sc[NB];
  uint32_t my_ptr = 0;
#pragma unroll
  // register sets that have not been filled yet hold a contig no anchor can have (and one different from the filler of
  // slots past the chunk end below), so "same contig and strand" alone rejects them: no `d <= i` / `i < n` tests per candidate
  for (int s = 0; s < NB; s++) { q[s] = r[s] = rt[s] = dpth[s] = 0; rc[s] = 0xFFFFFFFCu; sc[s] = 0; }
  for (uint32_t b0 = 0; b0 < nmax; b0 += GL) {
#pragma unroll
    for (int s = NB - 1; s > 0; s--) { q[s] = q[s - 1]; r[s] = r[s - 1]; rc[s] = rc[s - 1]; rt[s] = rt[s - 1]; dpth[s] = dpth[s - 1]; sc[s] = sc[s - 1]; }
    const uint32_t idx = b0 + gl;
    {
      AnchorRec x; x.qpos = 0; x.rpos = 0; x.rc = 0xFFFFFFFEu;            // impossible contig: never matches
      if (idx < n) {
        x = a[idx];
        if (onchip) s_word[idx] = idx << 8;
        else g_key[idx] = (unsigned long long)idx;
      }
      // the ref position is held NEGATED for reverse-strand anchors: two anchors can only chain on the same contig and
      // strand, and then (r' of the current) - (r' of the candidate) is the reference's strand-corrected ref gap directly
      q[0] = x.qpos; r[0] = (x.rc & 1u) ? (0u - x.rpos) : x.rpos; rc[0] = x.rc; sc[0] = 0; rt[0] = idx; dpth[0] = 1;
      my_ptr = idx;
    }
    __syncwarp();
#pragma unroll
    for (uint32_t m = 0; m < (uint32_t)GL; m++) {
      const uint32_t i = b0 + m;
      const uint32_t src = gbase | m;
      AnchorRec cur;
      cur.qpos = __shfl_sync(FULL, q[0], src);
      cur.rpos = __shfl_sync(FULL, r[0], src);
      cur.rc = __shfl_sync(FULL, rc[0], src);
      // The candidate in register set s is the predecessor at distance d = m - gl + GL * s.  Lanes that own an anchor of the
      // current block already scored (gl < m) use the sets 0 .. NE-1, the others 1 .. NE: the sets 1 .. NE-1 are common to all
      // lanes (no selects), only ONE "edge" candidate per lane is picked between set 0 and set NE.  The lane's best candidate
      // is kept as ONE key, (score - 1) << 5 | (31 - d): its maximum is the maximal score and, among those, the smallest
      // distance = largest j -- the reference's strict `>` while scanning j downward (src/chain.rs:853-880) -- and the group
      // arg-max is a single butterfly.  Keys of admissible candidates are > 0 (score >= 1, d <= 24).
      int32_t best = 0;
      const bool lo_set = gl < m;
      auto eval = [&](uint32_t qs, uint32_t rs, uint32_t rcs, int32_t scs, uint32_t d) {
        const uint32_t dq = cur.qpos - qs;
        const uint32_t dr = cur.rpos - rs;                                   // strand-corrected (see the load above)
        const uint32_t g = dr - dq;
        const bool ok = (FULLBAND || d <= band) & (rcs == cur.rc) & (dq - 1u < BP_CHAIN_BAND) & (dr - 1u < (uint32_t)MAX_LIN) &
                        (g + (uint32_t)MAX_GAP <= 2u * (uint32_t)MAX_GAP);
        const int32_t gi = (int32_t)g;
        const int32_t nsm1 = scs + (ANCHOR_SCORE - 1) - (gi < 0 ? -gi : gi);
        const int32_t key = (int32_t)(((uint32_t)nsm1 << 5) | (31u - d));
        best = max(best, ok ? key : 0);
      };
#pragma unroll
      for (int s2 = 1; s2 < NE; s2++) eval(q[s2], r[s2], rc[s2], sc[s2], m + (uint32_t)(GL * s2) - gl);
      eval(lo_set ? q[0] : q[NE], lo_set ? r[0] : r[NE], lo_set ? rc[0] : rc[NE], lo_set ? sc[0] : sc[NE],
           m - gl + (lo_set ? 0u : (uint32_t)(GL * NE)));
      int32_t kmax = best;
#pragma unroll
      for (int o = GL / 2; o > 0; o >>= 1) kmax = max(kmax, __shfl_xor_sync(FULL, kmax, o));
      const bool has = kmax > 0;
      const int32_t smax = (kmax >> 5) + 1;
      const uint32_t dwin = 31u - ((uint32_t)kmax & 31u);
      const uint32_t jw = i - dwin;                                          // only meaningful when has
      // winner's root / depth: owner lane = jw mod GL, set = block distance
      const int sidx = (int)(b0 >> LG) - (int)(jw >> LG);
      uint32_t rsel = rt[0], dsel = dpth[0];
#pragma unroll
      for (int s = 1; s < NB; s++) if (sidx == s) { rsel = rt[s]; dsel = dpth[s]; }
      const uint32_t wsrc = gbase | (jw & (uint32_t)(GL - 1));
      const uint32_t root_w = __shfl_sync(FULL, rsel, wsrc);
      const uint32_t depth_w = __shfl_sync(FULL, dsel, wsrc);
      const bool mine = has & (gl == m);
      sc[0] = mine ? smax : sc[0];
      rt[0] = mine ? root_w : rt[0];
      dpth[0] = mine ? depth_w + 1 : dpth[0];
      my_ptr = mine ? jw : my_ptr;
    }
    if (idx < n) {
      if (onchip) {
        if (rt[0] != idx) atomicMax(&s_word[rt[0]], ((uint32_t)sc[0] << 16) | (idx << 8) | (dpth[0] - 1));
      } else {
        g_depth[idx] = dpth[0];
        if (rt[0] != idx) atomicMax(&g_key[rt[0]], ((unsigned long long)(uint32_t)sc[0] << 32) | idx);
      }
      if (TAPS) { ws.score[a0 + idx] = sc[0]; ws.ptr[a0 + idx] = my_ptr; }
    }
  }
  __threadfence_block();
  __syncwarp();
  if (!live) return;
  const uint32_t p = ws.chunk_pair[c];
  const uint32_t qctg = ws.chunk_qctg[c];
  const uint32_t chunk_local_id = (uint32_t)(c - ws.pairCbase[p]);
  for (uint32_t i = gl; i < n; i += GL) {
    uint32_t b, score, num_anchors;
    if (onchip) {
      const uint32_t w = ((volatile uint32_t*)s_word)[i];
      b = (w >> 8) & 0xFFu; score = w >> 16; num_anchors = (w & 0xFFu) + 1;
      if (b == i) continue;                                          // singleton or not a root
    } else {
      if (((volatile uint32_t*)g_depth)[i] != 1) continue;          // not a root
      const unsigned long long key = ((volatile unsigned long long*)g_key)[i];
      b = (uint32_t)key; score = (uint32_t)(key >> 32);
      if (b == i) continue;                                          // singleton
      num_anchors = ((volatile uint32_t*)g_depth)[b];
    }
    if (num_anchors < MIN_ANCHORS || (int32_t)score < MIN_SCORE) continue;
    const AnchorRec f = a[i], l = a[b];
    uint32_t r0 = f.rpos < l.rpos ? f.rpos : l.rpos, r1 = f.rpos < l.rpos ? l.rpos : f.rpos;
    IntervalKey key5 = make_interval((int32_t)score, num_anchors, f.qpos, l.qpos, r0, r1, f.rc >> 1, qctg, chunk_local_id, f.rc & 1u);
    uint32_t slot2 = atomicAdd(&ws.pair_nint[p], 1u);
    ws.iv[ws.pairIbase[p] + slot2] = key5;
  }
}

// ------------------------------------------------------------------------------------------------------------
// K5: interval sort + greedy non-overlap selection, block per pair
// ------------------------------------------------------------------------------------------------------------
__device__ __forceinline__ bool interval_idx_before(uint32_t a, uint32_t b, unsigned long long ka, unsigned long long kb,
                                                    const IntervalKey* iv) {
  // a / b = interval indices (0xFFFFFFFF = padding, sorts last); ka / kb = their primary keys (score << 32 | num_anchors)
  if (a == 0xFFFFFFFFu) return false;
  if (b == 0xFFFFFFFFu) return true;
  if (ka != kb) return ka > kb;
  return interval_before(iv[a], iv[b]);   // rare: full derived-PartialOrd comparison on a primary-key tie
}

// bitonic sort of (primary key, index) pairs into the descending order of src/chain.rs:1012
__device__ void block_bitonic_sort_intervals(unsigned long long* key, uint32_t* idx, uint32_t npow2, const IntervalKey* iv) {
  for (uint32_t k = 2; k <= npow2; k <<= 1) {
    for (uint32_t j = k >> 1; j > 0; j >>= 1) {
      for (uint32_t i = threadIdx.x; i < npow2; i += blockDim.x) {
        uint32_t ixj = i ^ j;
        if (ixj > i) {
          uint32_t a = idx[i], b = idx[ixj];
          unsigned long long ka = key[i], kb = key[ixj];
          bool up = ((i & k) == 0);
          bool a_before_b = interval_idx_before(a, b, ka, kb, iv);
          bool swap = (a == b) ? false : (up ? !a_before_b : a_before_b);
          if (swap) { idx[i] = b; idx[ixj] = a; key[i] = kb; key[ixj] = ka; }
        }
      }
      __syncthreads();
    }
  }
}

constexpr uint32_t SEL_SMEM_MAX = 1024;   // intervals sorted / accepted in shared memory up to this many (power of two)
constexpr uint32_t SEL_CELL_SHIFT = 14;   // occupancy-bitmap cell = 16 kb
constexpr uint32_t SEL_MAP_BITS = 4096;

struct AccRec { uint32_t q0, q1, r0, r1, qctg, rctg; };

__device__ __forceinline__ uint32_t sel_cell_hash(uint32_t ctg, uint32_t cell) { return (cell + ctg * 0x9E37u) & (SEL_MAP_BITS - 1); }

constexpr uint32_t SEL_DEPS = 4;          // earlier overlapping candidates remembered per candidate (more -> full scan)

// Greedy non-overlap selection (src/chain.rs:1016-1095) is inherently ordered: candidate i is accepted iff its summed overlap
// with the ALREADY ACCEPTED intervals stays under half its length on both axes.  What is NOT ordered is finding out which
// earlier candidates can overlap it at all: every thread does that for its own candidates in parallel (n^2 / 2 interval
// tests per pair, shared-memory broadcasts), leaving a short dependency list per candidate; the ordered pass then only
// looks at the kept flags of those few predecessors (a candidate with more than SEL_DEPS of them scans the accepted list).
__global__ void __launch_bounds__(CT)
select_kernel(const PairDesc* __restrict__ pairs, ChainParams prm, Workspace ws) {
  __shared__ __align__(8) unsigned long long s_key[SEL_SMEM_MAX];   // sort keys; afterwards the dependency lists (u16 x SEL_DEPS)
  __shared__ uint32_t s_idx[SEL_SMEM_MAX];
  __shared__ AccRec s_cand[SEL_SMEM_MAX];       // candidates in sorted order
  __shared__ uint16_t s_accpos[SEL_SMEM_MAX];   // accepted candidates: their sorted positions
  __shared__ uint16_t s_cnt[SEL_SMEM_MAX];      // number of earlier candidates overlapping on either axis
  __shared__ uint8_t s_kept[SEL_SMEM_MAX];
  __shared__ uint32_t s_qmap[SEL_MAP_BITS / 32], s_rmap[SEL_MAP_BITS / 32];   // global-memory fallback only
  __shared__ uint32_t s_nacc;
  const unsigned FULL = 0xFFFFFFFFu;
  const uint32_t p = blockIdx.x;
  const uint32_t n = ws.pair_nint[p];
  if (n == 0) return;
  const uint64_t ib = ws.pairIbase[p];
  const IntervalKey* iv = ws.iv + ib;
  uint32_t npow2 = 1;
  while (npow2 < n) npow2 <<= 1;
  const bool in_smem = npow2 <= SEL_SMEM_MAX;
  // global fallback slices: iv_order has 4 slots per interval capacity, est_sorted-sized u64 scratch is not available here,
  // so the fallback keeps its primary keys in the iv_keys array (2 x u64 per interval capacity)
  uint32_t* idx = in_smem ? s_idx : (ws.iv_order + 4 * ib);
  unsigned long long* key = in_smem ? s_key : (ws.iv_keys + 2 * ib);
  for (uint32_t i = threadIdx.x; i < npow2; i += blockDim.x) {
    idx[i] = i < n ? i : 0xFFFFFFFFu;
    key[i] = i < n ? iv[i].k[0] : 0ull;
  }
  for (uint32_t i = threadIdx.x; i < SEL_MAP_BITS / 32; i += blockDim.x) { s_qmap[i] = 0; s_rmap[i] = 0; }
  __syncthreads();
  block_bitonic_sort_intervals(key, idx, npow2, iv);
  for (uint32_t i = threadIdx.x; i < n; i += blockDim.x) {
    const uint32_t ci = idx[i];
    ws.iv_order[4 * ib + npow2 + i] = ci;
    if (in_smem) {
      const IntervalKey c = iv[ci];
      AccRec x; x.q0 = iv_q0(c); x.q1 = iv_q1(c); x.r0 = iv_r0(c); x.r1 = iv_r1(c); x.qctg = iv_qctg(c); x.rctg = iv_rctg(c);
      s_cand[i] = x;
    }
  }
  if (threadIdx.x == 0) s_nacc = 0;
  __syncthreads();
  uint32_t* acc = ws.acc_list + ib;
  if (in_smem) {
    // ---- parallel: which earlier candidates overlap candidate i on the ref or on the query axis
    uint16_t* s_dep = (uint16_t*)s_key;
    for (uint32_t i = threadIdx.x; i < n; i += blockDim.x) {
      const AccRec c = s_cand[i];
      uint32_t cnt = 0;
      for (uint32_t j = 0; j < i; j++) {
        const AccRec x = s_cand[j];
        const bool ov = (x.rctg == c.rctg && x.r0 < c.r1 && c.r0 < x.r1) || (x.qctg == c.qctg && x.q0 < c.q1 && c.q0 < x.q1);
        if (ov) { if (cnt < SEL_DEPS) s_dep[i * SEL_DEPS + cnt] = (uint16_t)j; cnt++; }
      }
      s_cnt[i] = (uint16_t)min(cnt, 0xFFFFu);
    }
    __syncthreads();
    // ---- ordered pass, warp 0
    if (threadIdx.x < 32) {
      const uint32_t lane = threadIdx.x;
      uint32_t nacc = 0;
      for (uint32_t i = 0; i < n; i++) {
        const uint32_t cnt = s_cnt[i];
        bool ok = true;
        if (cnt != 0) {   // uniform
          const AccRec c = s_cand[i];
          uint32_t sum_r = 0, sum_q = 0;
          if (cnt <= SEL_DEPS) {
            if (lane < cnt) {
              const uint32_t j = s_dep[i * SEL_DEPS + lane];
              if (s_kept[j]) {
                const AccRec x = s_cand[j];
                // half-open overlap (bio IntervalTree::find), contribution = min(c.end - a.start, a.end - c.start) (src/chain.rs:1023-1086)
                if (x.rctg == c.rctg && x.r0 < c.r1 && c.r0 < x.r1) { const uint32_t u = c.r1 - x.r0, v = x.r1 - c.r0; sum_r = u < v ? u : v; }
                if (x.qctg == c.qctg && x.q0 < c.q1 && c.q0 < x.q1) { const uint32_t u = c.q1 - x.q0, v = x.q1 - c.q0; sum_q = u < v ? u : v; }
              }
            }
          } else {
            for (uint32_t a = lane; a < nacc; a += 32) {
              const AccRec x = s_cand[s_accpos[a]];
              if (x.rctg == c.rctg && x.r0 < c.r1 && c.r0 < x.r1) { const uint32_t u = c.r1 - x.r0, v = x.r1 - c.r0; sum_r += u < v ? u : v; }
              if (x.qctg == c.qctg && x.q0 < c.q1 && c.q0 < x.q1) { const uint32_t u = c.q1 - x.q0, v = x.q1 - c.q0; sum_q += u < v ? u : v; }
            }
          }
          sum_r = __reduce_add_sync(FULL, sum_r);
          sum_q = __reduce_add_sync(FULL, sum_q);
          // an overlapping interval always contributes > 0, so "no hit" == "sum is 0" (src/chain.rs:1042, 1072: OVERLAP_ORTHOLOGOUS_FRACTION)
          const bool ok_r = (sum_r == 0) || ((float)sum_r < (float)(c.r1 - c.r0) * 0.5f);
          const bool ok_q = (sum_q == 0) || ((float)sum_q < (float)(c.q1 - c.q0) * 0.5f);
          ok = ok_r && ok_q;
        }
        if (lane == 0) {
          const uint32_t ci = s_idx[i];
          s_kept[i] = ok ? 1 : 0;
          ws.iv_kept[ib + ci] = ok ? 1 : 0;
          if (ok) { acc[nacc] = ci; s_accpos[nacc] = (uint16_t)i; }
        }
        nacc += ok ? 1u : 0u;
        __syncwarp();
      }
      if (lane == 0) s_nacc = nacc;
    }
  } else if (threadIdx.x < 32) {
    // ---- more than SEL_SMEM_MAX intervals (huge / highly repetitive pairs): everything through global memory.  A 16 kb-cell
    //      occupancy bitmap per axis answers "cannot overlap anything accepted so far" in O(1) for most candidates.
    const uint32_t* order = ws.iv_order + 4 * ib + npow2;  // final sorted order lives after the sort scratch
    const uint32_t lane = threadIdx.x;
    uint32_t nacc = 0;
    for (uint32_t i = 0; i < n; i++) {
      const uint32_t ci = order[i];
      const IntervalKey c = iv[ci];
      const uint32_t q0 = iv_q0(c), q1 = iv_q1(c), r0 = iv_r0(c), r1 = iv_r1(c), qc = iv_qctg(c), rcg = iv_rctg(c);
      const uint32_t cq0 = q0 >> SEL_CELL_SHIFT, ncq = ((q1 - 1) >> SEL_CELL_SHIFT) - cq0 + 1;   // q0 < q1, r0 < r1 always
      const uint32_t cr0 = r0 >> SEL_CELL_SHIFT, ncr = ((r1 - 1) >> SEL_CELL_SHIFT) - cr0 + 1;
      bool need_scan = true;
      if (ncq <= 32 && ncr <= 32) {
        bool occ = false;
        if (lane < ncq) { uint32_t h = sel_cell_hash(qc, cq0 + lane); occ |= (s_qmap[h >> 5] >> (h & 31)) & 1u; }
        if (lane < ncr) { uint32_t h = sel_cell_hash(rcg, cr0 + lane); occ |= (s_rmap[h >> 5] >> (h & 31)) & 1u; }
        need_scan = __any_sync(FULL, occ);
      }
      bool ok = true;
      if (need_scan) {
        uint32_t sum_r = 0, hit_r = 0, sum_q = 0, hit_q = 0;
        for (uint32_t a = lane; a < nacc; a += 32) {
          uint32_t hr = 0, hq = 0;
          overlap_contrib(c, iv[acc[a]], &sum_r, &hr, &sum_q, &hq);
          hit_r |= hr ? 1u : 0u; hit_q |= hq ? 1u : 0u;
        }
        sum_r = __reduce_add_sync(FULL, sum_r);
        sum_q = __reduce_add_sync(FULL, sum_q);
        hit_r = __any_sync(FULL, hit_r) ? 1u : 0u;
        hit_q = __any_sync(FULL, hit_q) ? 1u : 0u;
        ok = overlap_accept(c, sum_r, hit_r, sum_q, hit_q);
      }
      if (ok) {
        if (lane == 0) acc[nacc] = ci;
        for (uint32_t t = lane; t < ncq; t += 32) { uint32_t h = sel_cell_hash(qc, cq0 + t); atomicOr(&s_qmap[h >> 5], 1u << (h & 31)); }
        for (uint32_t t = lane; t < ncr; t += 32) { uint32_t h = sel_cell_hash(rcg, cr0 + t); atomicOr(&s_rmap[h >> 5], 1u << (h & 31)); }
        nacc++;
      }
      if (lane == 0) ws.iv_kept[ib + ci] = ok ? 1 : 0;
      __syncwarp();
    }
    if (lane == 0) s_nacc = nacc;
  }
  __syncthreads();
  // accumulate the kept intervals into their chunks (src/chain.rs:204-251); all integer sums/min/max: order-free
  const uint32_t nacc = s_nacc;
  const uint64_t cbase = ws.pairCbase[p];
  const PairDesc pd = pairs[p];
  uint32_t my_sum = 0, my_cnt = 0;
  for (uint32_t a = threadIdx.x; a < nacc; a += blockDim.x) {
    const uint32_t ci = acc[a];
    const IntervalKey x = iv[ci];
    const uint64_t ch = cbase + iv_chunk(x);
    atomicAdd(&ws.acc_total[ch], iv_num_anchors(x));
    atomicMin(&ws.acc_rq0[ch], iv_q0(x));
    atomicMax(&ws.acc_rq1[ch], iv_q1(x));
    uint32_t span = pd.switched ? (iv_r1(x) - iv_r0(x)) : (iv_q1(x) - iv_q0(x));   // :223-237
    atomicAdd(&ws.acc_tbcq[ch], span + prm.k + 2 * prm.c);
    atomicAdd(&ws.acc_nint[ch], 1u);
    ws.iv_next[ib + ci] = atomicExch(&ws.chunk_head[ch], ci);
    my_sum += (iv_q1(x) - iv_q0(x)) + 2 * prm.c + prm.k;                            // :244-249 (overlap is always 0)
    my_cnt += 1;
  }
  if (my_cnt) { atomicAdd(&ws.pair_sumlen[p], my_sum); atomicAdd(&ws.pair_nchains[p], my_cnt); }
}

// ------------------------------------------------------------------------------------------------------------
// K6: per-chunk identity, one WARP per chunk: the lanes stride over the chunk's query seeds (coalesced), the chunk's kept
// intervals (1-3 as a rule) are read once into shared memory instead of being re-walked through global memory per seed
// ------------------------------------------------------------------------------------------------------------
constexpr int CS_WARPS = 8;        // warps per block
constexpr int CS_PER_WARP = 4;     // chunks handled by one warp, one after the other (32 chunks per block)
constexpr int CS_IV_MAX = 32;      // kept intervals of a chunk staged in shared memory; more are walked in global memory

// first index in [a, b) with pos[idx] > key (b if none), searched by the whole warp: 32 probes per round instead of one
__device__ __forceinline__ uint32_t warp_first_greater(const uint32_t* __restrict__ pos, uint32_t a, uint32_t b, int64_t key, uint32_t lane) {
  const unsigned FULL = 0xFFFFFFFFu;
  while (b - a > 32) {
    const uint32_t step = (b - a + 31) / 32;
    const uint32_t seg_b = min(a + (lane + 1) * step, b);          // this lane's segment is [a + lane * step, seg_b)
    const bool gt = (a + lane * step < b) && ((int64_t)pos[seg_b - 1] > key);
    const uint32_t m = __ballot_sync(FULL, gt);
    if (m == 0) return b;
    const uint32_t L = __ffs(m) - 1;
    const uint32_t na = a + L * step, nb = min(a + (L + 1) * step, b);
    a = na; b = nb;                                                 // the first greater element lies in segment L
  }
  const bool gt = (a + lane < b) && ((int64_t)pos[a + lane] > key);
  const uint32_t m = __ballot_sync(FULL, gt);
  return m ? a + __ffs(m) - 1 : b;
}

__global__ void __launch_bounds__(CS_WARPS * 32)
chunkstat_kernel(uint64_t n_chunks, const PairDesc* __restrict__ pairs, SetView s0, SetView s1,
                 const GenomeMeta* __restrict__ m0, const GenomeMeta* __restrict__ m1, ChainParams prm, Workspace ws,
                 uint32_t* __restrict__ dbg_counts) {
  __shared__ uint32_t s_start[CS_WARPS][CS_IV_MAX], s_stop[CS_WARPS][CS_IV_MAX];
  __shared__ uint32_t s_nseeds[CS_WARPS * CS_PER_WARP], s_numin[CS_WARPS * CS_PER_WARP], s_ul[CS_WARPS * CS_PER_WARP];
  const unsigned FULL = 0xFFFFFFFFu;
  const uint32_t lane = threadIdx.x & 31u, w = threadIdx.x >> 5;
  const uint64_t cblock = (uint64_t)blockIdx.x * (CS_WARPS * CS_PER_WARP);
  for (int k = 0; k < CS_PER_WARP; k++) {
    const uint32_t slot = w * CS_PER_WARP + k;
    const uint64_t c = cblock + slot;
    if (c >= n_chunks) break;                                  // warp-uniform
    const uint32_t p = ws.chunk_pair[c];
    const PairDesc pd = pairs[p];
    const SetView& Q = pd.qset ? s1 : s0;
    const GenomeMeta qm = (pd.qset ? m1 : m0)[pd.qg];
    const uint32_t n_int = ws.acc_nint[c], rq0 = ws.acc_rq0[c], rq1 = ws.acc_rq1[c];
    // seeds_in_chunk: counted query records of the chunk's contig with lo < pos <= hi
    const uint32_t ctg = ws.chunk_qctg[c];
    const uint32_t* cro = Q.ctg_rec_off + qm.ctg_off + qm.g;
    const uint32_t r0 = cro[ctg], r1 = cro[ctg + 1];
    const uint32_t* pos = Q.pv_pos + qm.seed_off;
    const int64_t lo = ws.chunk_lo[c], hi = ws.chunk_hi[c];
    const uint32_t first = warp_first_greater(pos, r0, r1, lo, lane);
    // a chunk spans <= 20 kb: its last seed is normally within a few hundred records of the first
    uint32_t cap = min(r1, first + 1024u);
    if (cap < r1 && (int64_t)pos[cap - 1] <= hi) cap = r1;
    const uint32_t last = warp_first_greater(pos, first, cap, hi, lane);   // [first, last)
    const uint32_t* cnt = ws.rec_cnt + (size_t)ws.tile_off[p] * (TILE / 32);   // the pair's "counted" bits
    const uint64_t ib = ws.pairIbase[p];
    const bool has_int = n_int > 0;
    // the chunk's kept intervals, padded by c on both sides (src/chain.rs:239-240), staged by lane 0
    uint32_t n_iv = 0, more = 0xFFFFFFFFu;
    __syncwarp();                                              // the previous chunk's readers of s_start / s_stop are done
    if (has_int) {
      if (lane == 0) {
        uint32_t i = ws.chunk_head[c];
        while (i != 0xFFFFFFFFu && n_iv < CS_IV_MAX) {
          const IntervalKey x = ws.iv[ib + i];
          const uint32_t q0 = iv_q0(x), q1 = iv_q1(x);
          s_start[w][n_iv] = padded_start(q0, prm.c);
          s_stop[w][n_iv] = q1 + prm.c;
          n_iv++;
          i = ws.iv_next[ib + i];
        }
        more = i;                                               // rest of the list (beyond CS_IV_MAX), walked in global memory
      }
      n_iv = __shfl_sync(FULL, n_iv, 0);
      more = __shfl_sync(FULL, more, 0);
      __syncwarp();
    }
    uint32_t n_seeds = 0, num_in = 0, upper_lower = 0;
    for (uint32_t t = first + lane; t < last; t += 32) {
      if (!((cnt[t >> 5] >> (t & 31u)) & 1u)) continue;
      n_seeds++;
      if (!has_int) continue;
      const uint32_t ps = pos[t];
      bool in = false;
      for (uint32_t i = 0; i < n_iv; i++) if (s_start[w][i] <= ps && ps <= s_stop[w][i]) { in = true; break; }
      for (uint32_t i = more; !in && i != 0xFFFFFFFFu; i = ws.iv_next[ib + i]) {
        const IntervalKey x = ws.iv[ib + i];
        if (seed_in_padded(ps, iv_q0(x), iv_q1(x), prm.c)) in = true;
      }
      if (in) num_in++;
      if (ps >= rq0 && ps <= rq1) upper_lower++;              // :322-328 with both spacing estimates 0
    }
    n_seeds = __reduce_add_sync(FULL, n_seeds);
    num_in = __reduce_add_sync(FULL, num_in);
    upper_lower = __reduce_add_sync(FULL, upper_lower);
    if (lane == 0) { s_nseeds[slot] = n_seeds; s_numin[slot] = num_in; s_ul[slot] = upper_lower; }
  }
  __syncthreads();
  // the per-chunk identity (two pow() calls) for the block's 32 chunks in parallel lanes
  if (threadIdx.x < CS_WARPS * CS_PER_WARP) {
    const uint64_t c = cblock + threadIdx.x;
    if (c < n_chunks) {
      ChunkAcc acc;
      acc.total_anchors = ws.acc_total[c]; acc.rq0 = ws.acc_rq0[c]; acc.rq1 = ws.acc_rq1[c];
      acc.tbcq = ws.acc_tbcq[c]; acc.n_int = ws.acc_nint[c];
      ws.chunk_nseeds[c] = s_nseeds[threadIdx.x];
      double est; uint32_t wgt;
      uint8_t valid = 0;
      bool filtered;
      if (chunk_estimate(acc, prm.c, prm.k, s_nseeds[threadIdx.x], s_numin[threadIdx.x], s_ul[threadIdx.x], &est, &wgt, &filtered)) {
        ws.chunk_est[c] = est; ws.chunk_w[c] = wgt; valid = filtered ? 3 : 1;   // 3: the putative-ANI filter applied
        if (prm.c >= 200) atomicAdd(&ws.pair_tqb_ns[ws.chunk_pair[c]], acc.rq1 - acc.rq0 + 2 * prm.c + prm.k);  // !sensitive_af (:261-264)
      }
      ws.chunk_valid[c] = valid;
      if (dbg_counts) {                                        // debug runs: the warp-reduced counts and the filter decision
        dbg_counts[3 * c] = s_numin[threadIdx.x]; dbg_counts[3 * c + 1] = s_ul[threadIdx.x]; dbg_counts[3 * c + 2] = filtered ? 1u : 0u;
      }
    }
  }
}

// test use (sk_debug_chunk_estimate): chunk_estimate on given accumulations and counts, 8 x u32 per chunk
__global__ void debug_chunk_estimate_kernel(uint64_t n, const uint32_t* __restrict__ in, uint32_t c, uint32_t k, double* est,
                                            uint32_t* weight, uint32_t* valid) {
  const uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const uint32_t* x = in + 8 * i;
  ChunkAcc acc;
  acc.total_anchors = x[0]; acc.rq0 = x[1]; acc.rq1 = x[2]; acc.tbcq = x[3]; acc.n_int = x[4];
  double e = 0.; uint32_t w = 0; bool f = false;
  const bool ok = chunk_estimate(acc, c, k, x[5], x[6], x[7], &e, &w, &f);
  est[i] = ok ? e : 0.; weight[i] = ok ? w : 0u; valid[i] = ok ? (f ? 3u : 1u) : 0u;
}

// ------------------------------------------------------------------------------------------------------------
// K7: final statistics, block per pair
// ------------------------------------------------------------------------------------------------------------
struct EstKey { double e; uint32_t w; };
__device__ __forceinline__ bool est_less(double ea, uint32_t wa, double eb, uint32_t wb) {  // (f64, usize) tuple order (:414)
  if (ea != eb) return ea < eb;
  return wa < wb;
}

constexpr int FT = 128;                      // >= BOOT_ITERS: one replicate per thread
constexpr uint32_t FIN_SMEM_MAX = 1024;
constexpr uint32_t GBDT_TREES = SK_GBDT_C125_NTREES;   // one tree per thread
static_assert(SK_GBDT_C125_NTREES == SK_GBDT_C200_NTREES, "both models have the same number of trees");
static_assert(FT >= (int)BOOT_ITERS, "final_kernel runs one bootstrap replicate per thread");

__global__ void __launch_bounds__(FT)
final_kernel(const PairDesc* __restrict__ pairs, const GenomeMeta* __restrict__ m0, const GenomeMeta* __restrict__ m1,
             ChainParams prm, Workspace ws, sk_ani_result* __restrict__ out, int force_redo) {
  __shared__ double s_e[FIN_SMEM_MAX];
  __shared__ uint32_t s_w[FIN_SMEM_MAX];
  __shared__ uint64_t s_cum[FIN_SMEM_MAX];
  __shared__ uint32_t s_n;
  __shared__ double s_boot[BOOT_ITERS];
  __shared__ double s_ci[2];
  __shared__ uint16_t s_guide[GUIDE_BUCKETS];
  __shared__ float s_term[GBDT_TREES];
  __shared__ float s_x[5];
  __shared__ int s_do_reg;
  __shared__ uint32_t s_reject;
  __shared__ double s_final, s_std;
  __shared__ uint64_t s_pool;
  const uint32_t p = blockIdx.x;
  const PairDesc pd = pairs[p];
  const GenomeMeta refm = m0[pd.ref_idx];     // the call's ref / query sketches (un-switched, src/chain.rs:477-484)
  const GenomeMeta qrym = m1[pd.query_idx];
  sk_ani_result r;
  memset(&r, 0, sizeof(r));
  r.ref_id = pd.ref_idx; r.query_id = pd.query_idx;
  const uint64_t cb = ws.pairCbase[p];
  const uint32_t nc = ws.pairC[p];
  // compact valid chunk estimates
  double* ge = (nc <= FIN_SMEM_MAX) ? s_e : ws.est_sorted + 4 * cb;
  uint32_t* gw = (nc <= FIN_SMEM_MAX) ? s_w : ws.w_sorted + 4 * cb;
  if (threadIdx.x == 0) s_n = 0;
  __syncthreads();
  uint32_t npow2 = 1;
  while (npow2 < nc) npow2 <<= 1;
  // deterministic compaction is unnecessary: the list is sorted next (ties are exact duplicates)
  for (uint32_t i = threadIdx.x; i < nc; i += blockDim.x) {
    if (ws.chunk_valid[cb + i]) {
      uint32_t slot = atomicAdd(&s_n, 1u);
      ge[slot] = ws.chunk_est[cb + i]; gw[slot] = ws.chunk_w[cb + i];
    }
  }
  __syncthreads();
  const uint32_t n = s_n;
  const uint32_t num_chains = ws.pair_nchains[p];
  if (n == 0 || num_chains == 0) {                       // src/chain.rs:416-420: default result with ani = NaN
    if (threadIdx.x == 0) { r.ani = nanf(""); out[p] = r; }
    return;
  }
  uint32_t np2 = 1;
  while (np2 < n) np2 <<= 1;
  for (uint32_t i = n + threadIdx.x; i < np2; i += blockDim.x) { ge[i] = INFINITY; gw[i] = 0xFFFFFFFFu; }
  __syncthreads();
  for (uint32_t k = 2; k <= np2; k <<= 1) {
    for (uint32_t j = k >> 1; j > 0; j >>= 1) {
      for (uint32_t i = threadIdx.x; i < np2; i += blockDim.x) {
        uint32_t ixj = i ^ j;
        if (ixj > i) {
          bool up = ((i & k) == 0);
          bool a_lt_b = est_less(ge[i], gw[i], ge[ixj], gw[ixj]);
          bool b_lt_a = est_less(ge[ixj], gw[ixj], ge[i], gw[i]);
          bool swap = up ? b_lt_a : a_lt_b;
          if (swap) { double te = ge[i]; ge[i] = ge[ixj]; ge[ixj] = te; uint32_t tw = gw[i]; gw[i] = gw[ixj]; gw[ixj] = tw; }
        }
      }
      __syncthreads();
    }
  }
  // sequential part (exact left-to-right f64 sums as the reference): thread 0
  if (threadIdx.x == 0) {
    uint64_t total_mult = 0;
    for (uint32_t i = 0; i < n; i++) total_mult += gw[i];
    double lower, upper;
    trim_fractions(prm.median != 0, prm.robust != 0, &lower, &upper);
    uint32_t lower_i, upper_i;
    trim_bounds(gw, n, total_mult, lower, upper, &lower_i, &upper_i);
    s_final = trimmed_mean(ge, gw, lower_i, upper_i);
    s_std = pop_std(ge, n);
    s_reject = force_redo ? 1u : 0u;
    s_pool = total_mult;
  }
  __syncthreads();
  // bootstrap (src/chain.rs:57-86): BOOT_ITERS replicates x n draws from the weight-expanded pool; replicate r uses draws
  // [r*n, (r+1)*n) of the WyRand stream, each replicate summed sequentially by one thread.
  double ci_lo = 0., ci_hi = 1.;
  if (boot_enabled(n)) {
    const uint64_t pool = s_pool;
    // inclusive running weights for the idx -> estimate lookup, built once
    uint64_t* cum = (nc <= FIN_SMEM_MAX) ? s_cum : (uint64_t*)(ws.est_sorted + 4 * cb + npow2);  // global scratch: 8 B per chunk available
    if (threadIdx.x == 0) {
      uint64_t run = 0;
      for (uint32_t i = 0; i < n; i++) { run += gw[i]; cum[i] = run; }
    }
    __syncthreads();
    const uint32_t gshift = guide_shift(pool);
    const uint32_t nbuck = guide_buckets(pool, gshift);
    for (uint32_t bk = threadIdx.x; bk < nbuck; bk += blockDim.x) s_guide[bk] = guide_entry(cum, n, bk, gshift);
    __syncthreads();
    if (threadIdx.x < BOOT_ITERS) {
      bool rej;
      double m;
      if (nc <= FIN_SMEM_MAX && n < GUIDE_MAX_N) m = boot_replicate<true>(s_cum, s_e, n, pool, s_guide, gshift, threadIdx.x, &rej);   // shared-memory operands (LDS), the common case
      else if (n < GUIDE_MAX_N) m = boot_replicate<true>(cum, ge, n, pool, s_guide, gshift, threadIdx.x, &rej);
      else m = boot_replicate<false>(cum, ge, n, pool, nullptr, 0, threadIdx.x, &rej);                 // 65535 estimates or more: plain search
      s_boot[threadIdx.x] = m;
      if (rej) atomicOr(&s_reject, 1u);
    }
    __syncthreads();
    // a Lemire rejection shifts the stream: redo sequentially (probability ~ n * 100 * pool / 2^64)
    if (threadIdx.x == 0 && s_reject) boot_redo(cum, ge, n, pool, s_boot);
    __syncthreads();
    // order statistics of the replicate means (src/chain.rs:80-85 sorts them): every thread ranks its own value instead of
    // one thread sorting serially
    if (threadIdx.x < BOOT_ITERS) {
      const uint32_t rank = boot_rank(s_boot, threadIdx.x);
      if (rank == CI_LO_RANK) s_ci[0] = s_boot[threadIdx.x];
      if (rank == CI_HI_RANK) s_ci[1] = s_boot[threadIdx.x];
    }
    __syncthreads();
    ci_lo = s_ci[0]; ci_hi = s_ci[1];
  }
  if (threadIdx.x == 0) {
    double final_ani = s_final;
    const uint32_t sumlen = ws.pair_sumlen[p];
    const uint32_t tqb = (prm.c < 200) ? sumlen : ws.pair_tqb_ns[p];      // sensitive_af (:183-190, 244-247, 261-264)
    const double covered_query = covered_frac(tqb, qrym.total_len), covered_ref = covered_frac(tqb, refm.total_len);
    if (af_cut(covered_query, covered_ref, prm.frac_cover_cutoff, prm.both_frac_cover_cutoff)) final_ani = -1.;
    r.ani = (float)final_ani;
    r.af_query = (float)covered_query; r.af_ref = (float)covered_ref;
    r.ci_lower = (float)ci_lo; r.ci_upper = (float)ci_hi; r.std = (float)s_std;
    r.q10_q = (float)qrym.q10; r.q50_q = (float)qrym.q50; r.q90_q = (float)qrym.q90;
    r.q10_r = (float)refm.q10; r.q50_r = (float)refm.q50; r.q90_r = (float)refm.q90;
    r.num_contigs_q = qrym.n_ctg; r.num_contigs_r = refm.n_ctg;
    r.avg_chain_int_len = sumlen / num_chains;            // u32 division (:421)
    r.total_bases_covered = tqb;
    // learned-ANI regression (src/regression.rs:30-64): features now, the 195 trees are walked by all threads below
    s_do_reg = 0;
    if (prm.model >= 0 && regress_gate(r.ani, r.total_bases_covered)) {
      regress_features(r.ani, r.std, r.q50_q, r.q90_q, r.q50_r, r.q90_r, r.avg_chain_int_len, s_x);
      s_do_reg = 1;
    }
  }
  __syncthreads();
  if (s_do_reg) {   // uniform
    // gbdt_eval with the per-tree terms (independent) one per thread, then summed in tree order by thread 0
    const unsigned char* feat = c_gbdt_feat[prm.model];
    const float* thr = c_gbdt_thr[prm.model];
    const float* leaf = c_gbdt_leaf[prm.model];
    const float shrink = c_gbdt_shrink[prm.model];
    for (uint32_t t = threadIdx.x; t < GBDT_TREES; t += blockDim.x) s_term[t] = gbdt_tree_term(feat, thr, leaf, (int)t, shrink, s_x);
    __syncthreads();
    if (threadIdx.x == 0) {
      float pred = c_gbdt_bias[prm.model];
      for (uint32_t t = 0; t < GBDT_TREES; t++) pred = fadd_rn(pred, s_term[t]);
      regress_apply(pred, &r.ani, &r.ci_lower, &r.ci_upper);
    }
  }
  if (threadIdx.x == 0) out[p] = r;
}

// ------------------------------------------------------------------------------------------------------------
// K8 (sk_chain_pairs_mappings only): the kept intervals of every pair as sorted sk_mapping records
// ------------------------------------------------------------------------------------------------------------
constexpr int MAP_SCAN_T = 256;
constexpr uint32_t MAP_SMEM_MAX = 512;   // records of a pair sorted in shared memory; a pair with more sorts in global memory

// map_base[0..B] = exclusive prefix of pair_nchains (the kept intervals of each pair), one block
__global__ void __launch_bounds__(MAP_SCAN_T)
mapping_scan_kernel(uint32_t B, const uint32_t* __restrict__ nchains, uint64_t* __restrict__ map_base) {
  using Scan = cub::BlockScan<uint64_t, MAP_SCAN_T>;
  __shared__ typename Scan::TempStorage tmp;
  __shared__ uint64_t s_carry;
  if (threadIdx.x == 0) s_carry = 0;
  __syncthreads();
  for (uint32_t i0 = 0; i0 < B; i0 += MAP_SCAN_T) {
    const uint32_t i = i0 + threadIdx.x;
    uint64_t ex, tot;
    Scan(tmp).ExclusiveSum(i < B ? (uint64_t)nchains[i] : 0ull, ex, tot);
    if (i < B) map_base[i] = s_carry + ex;
    __syncthreads();
    if (threadIdx.x == 0) s_carry += tot;
    __syncthreads();
  }
  if (threadIdx.x == 0) map_base[B] = s_carry;
}

// Block per pair: the pair's kept intervals (acc_list, in selection order) become records joined to their chunk's estimate
// (mapping_record), are bitonic-sorted by mapping_before through an index array and written to out[map_base[p] ..).  Up to
// MAP_SMEM_MAX records the records and indices live in shared memory; beyond, in the pair's slices of stage (one record per
// kept interval) and gidx (two indices per kept interval >= the padded power of two).
__global__ void __launch_bounds__(CT)
mapping_emit_kernel(const PairDesc* __restrict__ pairs, Workspace ws, const uint64_t* __restrict__ map_base,
                    sk_mapping* __restrict__ stage, uint32_t* __restrict__ gidx, sk_mapping* __restrict__ out) {
  __shared__ sk_mapping s_rec[MAP_SMEM_MAX];
  __shared__ uint32_t s_idx[MAP_SMEM_MAX];
  const uint32_t p = blockIdx.x;
  const uint64_t base = map_base[p];
  const uint32_t n = (uint32_t)(map_base[p + 1] - base);
  if (n == 0) return;
  uint32_t npow2 = 1;
  while (npow2 < n) npow2 <<= 1;
  const bool in_smem = npow2 <= MAP_SMEM_MAX;
  sk_mapping* rec = in_smem ? s_rec : stage + base;
  uint32_t* idx = in_smem ? s_idx : gidx + 2 * base;
  const uint64_t ib = ws.pairIbase[p], cb = ws.pairCbase[p];
  const bool sw = pairs[p].switched != 0;
  const uint32_t NONE = 0xFFFFFFFFu;
  for (uint32_t a = threadIdx.x; a < npow2; a += blockDim.x) {
    if (a < n) {
      const IntervalKey x = ws.iv[ib + ws.acc_list[ib + a]];
      const uint64_t ch = cb + iv_chunk(x);
      const uint8_t v = ws.chunk_valid[ch];
      rec[a] = mapping_record(x, sw, v ? ws.chunk_est[ch] : 0., v ? ws.chunk_w[ch] : 0u, v);
    }
    idx[a] = a < n ? a : NONE;   // padding sorts last
  }
  __syncthreads();
  for (uint32_t k = 2; k <= npow2; k <<= 1) {
    for (uint32_t j = k >> 1; j > 0; j >>= 1) {
      for (uint32_t i = threadIdx.x; i < npow2; i += blockDim.x) {
        const uint32_t ixj = i ^ j;
        if (ixj > i) {
          const uint32_t a = idx[i], b = idx[ixj];
          const bool b_lt_a = b != NONE && (a == NONE || mapping_before(rec[b], rec[a]));
          const bool a_lt_b = a != NONE && (b == NONE || mapping_before(rec[a], rec[b]));
          if ((i & k) == 0 ? b_lt_a : a_lt_b) { idx[i] = b; idx[ixj] = a; }
        }
      }
      __syncthreads();
    }
  }
  for (uint32_t i = threadIdx.x; i < n; i += blockDim.x) out[base + i] = rec[idx[i]];
}

__global__ void chunk_size_kernel(uint64_t n, Workspace ws) {
  uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  ws.chunk_size[i] = (uint32_t)(ws.chunk_first[i + 1] - ws.chunk_first[i]);
  ws.chunk_id[i] = (uint32_t)i;
}

__global__ void init_chunk_acc_kernel(uint64_t n, Workspace ws) {
  uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  ws.acc_total[i] = 0; ws.acc_rq0[i] = 0xFFFFFFFFu; ws.acc_rq1[i] = 0; ws.acc_tbcq[i] = 0; ws.acc_nint[i] = 0;
  ws.chunk_head[i] = 0xFFFFFFFFu;
}

// ------------------------------------------------------------------------------------------------------------
// host
// ------------------------------------------------------------------------------------------------------------
static bool g_tables_uploaded[64] = {false};
static std::mutex g_tables_mu;

// constant-memory GBDT tables, once per device.  Several contexts (the pipelined worker, sk_triangle_multi's per-device
// threads) may get here concurrently: serialised, and the device is synchronised before the flag is published so that
// no kernel on a non-blocking stream can run ahead of the upload.
static int upload_tables(sk_ctx* ctx) {
  std::lock_guard<std::mutex> lk(g_tables_mu);
  if (ctx->device < 64 && g_tables_uploaded[ctx->device]) return SK_OK;
  static float thr[2][1365], leaf[2][1560], shrink[2], bias[2];
  static unsigned char feat[2][1365];
  auto b2f = [](uint32_t b) { float f; memcpy(&f, &b, 4); return f; };
  for (int i = 0; i < 1365; i++) {
    feat[0][i] = tables::SK_GBDT_C125_FEAT[i]; feat[1][i] = tables::SK_GBDT_C200_FEAT[i];
    thr[0][i] = b2f(tables::SK_GBDT_C125_THR[i]); thr[1][i] = b2f(tables::SK_GBDT_C200_THR[i]);
  }
  for (int i = 0; i < 1560; i++) { leaf[0][i] = b2f(tables::SK_GBDT_C125_LEAF[i]); leaf[1][i] = b2f(tables::SK_GBDT_C200_LEAF[i]); }
  shrink[0] = b2f(SK_GBDT_C125_SHRINK_BITS); shrink[1] = b2f(SK_GBDT_C200_SHRINK_BITS);
  bias[0] = b2f(SK_GBDT_C125_BIAS_BITS); bias[1] = b2f(SK_GBDT_C200_BIAS_BITS);
  SK_CUDA(cudaMemcpyToSymbol(c_gbdt_feat, feat, sizeof(feat)));
  SK_CUDA(cudaMemcpyToSymbol(c_gbdt_thr, thr, sizeof(thr)));
  SK_CUDA(cudaMemcpyToSymbol(c_gbdt_leaf, leaf, sizeof(leaf)));
  SK_CUDA(cudaMemcpyToSymbol(c_gbdt_shrink, shrink, sizeof(shrink)));
  SK_CUDA(cudaMemcpyToSymbol(c_gbdt_bias, bias, sizeof(bias)));
  SK_CUDA(cudaDeviceSynchronize());
  if (ctx->device < 64) g_tables_uploaded[ctx->device] = true;
  return SK_OK;
}

static SetView view_of(const sk_sketch_set* s) {
  SetView v;
  v.pv_kmer = s->pv_kmer; v.pv_pos = s->pv_pos; v.pv_cc = s->pv_cc; v.pv_mult = s->pv_mult;
  v.kv_pos = s->kv_pos; v.kv_cc = s->kv_cc; v.ukmer = s->ukmer; v.ustart = s->ustart; v.ctg_rec_off = s->ctg_rec_off; v.ubucket = s->ubucket; v.htab = s->htab;
  return v;
}

static void build_meta(const sk_sketch_set* s, std::vector<GenomeMeta>& out) {
  out.resize(s->G);
  std::vector<uint32_t> tmp;
  for (uint32_t g = 0; g < s->G; g++) {
    GenomeMeta& m = out[g];
    m.seed_off = s->seed_off[g]; m.uk_off = s->uk_off[g]; m.ctg_off = s->ctg_off[g];
    m.n_rec = (uint32_t)(s->seed_off[g + 1] - s->seed_off[g]);
    m.n_uk = (uint32_t)(s->uk_off[g + 1] - s->uk_off[g]);
    m.n_ctg = (uint32_t)(s->ctg_off[g + 1] - s->ctg_off[g]);
    m.g = g; m.total_len = s->total_len[g]; m.pad = 0;
    m.ht_off = s->ht_off.empty() ? 0 : s->ht_off[g];
    m.ht_cap = s->ht_off.empty() ? 0 : (uint32_t)(s->ht_off[g + 1] - s->ht_off[g]);
    tmp.assign(s->ctg_len.begin() + s->ctg_off[g], s->ctg_len.begin() + s->ctg_off[g + 1]);
    uint64_t max_chunks = 0;      // a contig-local chunk index never exceeds need < len / FRAGMENT_LENGTH
    for (uint32_t len : tmp) max_chunks += (len + (uint64_t)FRAGMENT_LENGTH - 1) / FRAGMENT_LENGTH;
    m.max_chunks = (uint32_t)std::min<uint64_t>(max_chunks, 0xFFFFFFFFu);
    std::sort(tmp.begin(), tmp.end());
    size_t n = tmp.size();
    m.q10 = n ? tmp[n * 10 / 100] : 0; m.q50 = n ? tmp[n * 50 / 100] : 0; m.q90 = n ? tmp[n * 90 / 100] : 0;  // src/chain.rs:519-526
  }
}

// role selection of get_anchors (src/chain.rs:625-661) + switch_qr (:15-26), in f64 exactly as the reference
static bool pair_switched(const sk_sketch_set* refs, uint32_t r, const sk_sketch_set* qs, uint32_t q, bool same_set) {
  auto mean_len = [](const sk_sketch_set* s, uint32_t g) {
    double sum = 0;
    for (uint64_t c = s->ctg_off[g]; c < s->ctg_off[g + 1]; c++) sum += (double)s->ctg_len[c];
    return sum / (double)(s->ctg_off[g + 1] - s->ctg_off[g]);
  };
  double mean_q = mean_len(qs, q), mean_r = mean_len(refs, r);
  double qp, rp;
  if (qs->total_len[q] > 100000 && refs->total_len[r] > 100000) {
    qp = (double)(qs->mk_off[q + 1] - qs->mk_off[q]) * (double)qs->sp.c;
    rp = (double)(refs->mk_off[r + 1] - refs->mk_off[r]) * (double)refs->sp.c;
  } else {
    qp = (double)qs->total_len[q]; rp = (double)refs->total_len[r];
  }
  double score_query = qp * std::min(mean_q, 300000.);
  double score_ref = rp * std::min(mean_r, 300000.);
  if (score_query == score_ref) {
    uint64_t rq = qs->name_rank[q] + ((same_set || qs->ranks_user_set) ? 0 : refs->G), rr = refs->name_rank[r];
    return rq > rr;  // query_file_name > ref_file_name
  }
  return score_query > score_ref;
}

struct BatchBuffers {  // grow-only device buffers reused across batches
  std::vector<std::pair<void**, size_t>> reg;
};

template <typename T>
static int ensure(sk_ctx* ctx, T** p, size_t* cap, size_t need) {
  if (need <= *cap && *p) return SK_OK;
  // grow-only, kept for the life of the context: plain cudaMalloc (outside the stream-ordered pool, whose reuse of
  // multi-GB blocks of varying size proved erratic); growth happens only while the workload is still getting larger
  if (*p) SK_CUDA(cudaFree(*p));
  *p = nullptr;
  size_t n = std::max<size_t>(need + need / 4, 1024);
  SK_CUDA(cudaMalloc((void**)p, n * sizeof(T)));
  *cap = n;
  return SK_OK;
}

struct ChainScratch {
  Workspace ws{};
  size_t cap_rec = 0, cap_pair = 0, cap_anc = 0, cap_chunk = 0, cap_iv = 0;
  size_t c_hit = 0, c_tile_hits = 0, c_rec_cnt = 0, c_tile_off = 0;
  size_t c_stg_first = 0, c_stg_qctg = 0, c_stg_lo = 0, c_stg_hi = 0;
  size_t c_pairA = 0, c_pairC = 0, c_pairAbase = 0, c_pairCbase = 0, c_pairIbase = 0, c_pair_nint = 0, c_pair_sumlen = 0,
         c_pair_nchains = 0, c_pair_tqb = 0;
  size_t c_anc = 0, c_score = 0, c_ptr = 0, c_rootkey = 0, c_depth = 0;
  size_t c_chunk_size = 0, c_chunk_size_sorted = 0, c_chunk_id = 0, c_chunk_perm = 0, c_sort_tmp = 0;
  uint8_t* sort_tmp = nullptr;
  uint32_t* dbg_counts = nullptr; size_t c_dbg_counts = 0;   // debug runs: chunkstat_kernel's num_in, upper_lower, filtered
  size_t c_chunk_first = 0, c_chunk_pair = 0, c_chunk_qctg = 0, c_chunk_lo = 0, c_chunk_hi = 0, c_acc_total = 0, c_acc_rq0 = 0,
         c_acc_rq1 = 0, c_acc_tbcq = 0, c_acc_nint = 0, c_chunk_head = 0, c_chunk_est = 0, c_chunk_w = 0, c_chunk_valid = 0, c_chunk_nseeds = 0;
  size_t c_iv = 0, c_iv_keys = 0, c_iv_order = 0, c_iv_kept = 0, c_iv_next = 0, c_acc_list = 0, c_est_sorted = 0, c_w_sorted = 0;
  PairDesc* d_pairs = nullptr; size_t c_pairs = 0;
  sk_ani_result* d_out = nullptr; size_t c_out = 0;
  // mapping runs only: per-pair record offsets, the sorted records, and the global-memory sort's records and indices
  uint64_t* map_base = nullptr; size_t c_map_base = 0;
  sk_mapping *map_out = nullptr, *map_stage = nullptr; size_t c_map_out = 0, c_map_stage = 0;
  uint32_t* map_idx = nullptr; size_t c_map_idx = 0;
  sk_mapping* h_map = nullptr; size_t c_h_map = 0;   // pinned staging of a batch's records on their way to the host
  GenomeMeta *d_m0 = nullptr, *d_m1 = nullptr;
  size_t c_m0 = 0, c_m1 = 0;
  void free_all() {
    void* ptrs[] = {ws.chunk_size, ws.chunk_size_sorted, ws.chunk_id, ws.chunk_perm, sort_tmp, dbg_counts, ws.hit, ws.tile_hits, ws.rec_cnt, ws.tile_off, ws.stg_first, ws.stg_qctg, ws.stg_lo, ws.stg_hi,
                    ws.pairA, ws.pairC, ws.pairAbase, ws.pairCbase, ws.pairIbase, ws.pair_nint, ws.pair_sumlen, ws.pair_nchains, ws.pair_tqb_ns, ws.anc,
                    ws.score, ws.ptr, ws.rootkey, ws.depth, ws.chunk_first, ws.chunk_pair, ws.chunk_qctg, ws.chunk_lo, ws.chunk_hi,
                    ws.acc_total, ws.acc_rq0, ws.acc_rq1, ws.acc_tbcq, ws.acc_nint, ws.chunk_head, ws.chunk_est, ws.chunk_w, ws.chunk_valid,
                    ws.chunk_nseeds, ws.iv, ws.iv_keys, ws.iv_order, ws.iv_kept, ws.iv_next, ws.acc_list, ws.est_sorted, ws.w_sorted, d_pairs, d_out, d_m0, d_m1,
                    map_base, map_out, map_stage, map_idx};
    for (void* p : ptrs) if (p) cudaFree(p);
    if (h_map) cudaFreeHost(h_map);
  }
};

struct HostPair { uint32_t ref, query; };

// the mappings of a call, collected batch by batch in pair order: count[i] records of pair i, all pairs' n records in recs
// (malloc'd: handed to the caller as is)
struct MapOut {
  std::vector<uint64_t> count;
  sk_mapping* recs = nullptr;
  size_t n = 0, cap = 0;
  ~MapOut() { free(recs); }
};

// dp_group_kernel's instantiation for the band: FULLBAND when the band fills the lanes' register sets exactly, and then the
// 25-block register cap unless SK_DP_MINB=1.  TAPS only adds the score / pointer stores.
template <bool TAPS, int GL, int NE>
static int launch_dp_group(sk_ctx* ctx, uint32_t grid, uint64_t TC, const ChainParams& prm, const Workspace& ws, int dp_minb) {
  cudaStream_t st = ctx->stream;
  if (prm.band == GL * NE && dp_minb > 1) SK_LAUNCH(ctx, "dp_kernel", (dp_group_kernel<TAPS, GL, NE, true, 25><<<grid, 32, 0, st>>>(TC, prm, ws)));
  else if (prm.band == GL * NE) SK_LAUNCH(ctx, "dp_kernel", (dp_group_kernel<TAPS, GL, NE, true, 1><<<grid, 32, 0, st>>>(TC, prm, ws)));
  else SK_LAUNCH(ctx, "dp_kernel", (dp_group_kernel<TAPS, GL, NE, false, 1><<<grid, 32, 0, st>>>(TC, prm, ws)));
  return SK_OK;
}

// The chain back end's DP and interval selection on the workspace as chunk_compact_kernel / init_chunk_acc_kernel leave it
// (TC > 0 chunks of B pairs): the DP instantiation the band (and the SK_DP_* A/B hooks) choose, then select_kernel.  run_batch
// and the test entries sk_debug_chain_anchors (dp) / sk_debug_select_intervals (!dp, intervals given) all launch through here.
// taps: the DP also stores the per-anchor scores and pointers.
static int launch_dp_select(sk_ctx* ctx, ChainScratch& S, uint32_t B, uint64_t TC, const ChainParams& prm, bool dp, bool taps) {
  cudaStream_t st = ctx->stream;
  Workspace& ws = S.ws;
  if (dp) {
    const uint32_t grid = (uint32_t)TC;
    const uint32_t nb = prm.band / 32 + 2;   // register sets per lane: current block + ceil(band / 32) earlier ones
#define DP_LAUNCH(NBV)                                                                                       \
  if (taps) SK_LAUNCH(ctx, "dp_kernel", (dp_warp_kernel<NBV, true><<<grid, 32, 0, st>>>(TC, prm, ws)));       \
  else SK_LAUNCH(ctx, "dp_kernel", (dp_warp_kernel<NBV, false><<<grid, 32, 0, st>>>(TC, prm, ws)));
    if (prm.band <= 24 && getenv("SK_DP_WARP") == nullptr) {   // 4 chunks per warp, 8 lanes each
      const int dp_gl = getenv("SK_DP_GL") ? atoi(getenv("SK_DP_GL")) : 4;   // lanes per chunk: 4 (default, faster in A/B runs) or 8
      const int dp_minb = getenv("SK_DP_MINB") ? atoi(getenv("SK_DP_MINB")) : 25;   // register cap: 72 registers = 28 resident warps per SM (A/B: 1 = uncapped)
      const uint32_t gw = dp_gl == 4 ? 8 : 4;
      const uint32_t g4 = (uint32_t)((TC + gw - 1) / gw);
      // group chunks of similar size: sort chunk ids by descending anchor count (cub radix sort, ~0.1 ms per batch)
      SK_TRY(ensure(ctx, &ws.chunk_size, &S.c_chunk_size, TC)); SK_TRY(ensure(ctx, &ws.chunk_size_sorted, &S.c_chunk_size_sorted, TC));
      SK_TRY(ensure(ctx, &ws.chunk_id, &S.c_chunk_id, TC)); SK_TRY(ensure(ctx, &ws.chunk_perm, &S.c_chunk_perm, TC));
      chunk_size_kernel<<<(uint32_t)((TC + 255) / 256), 256, 0, st>>>(TC, ws); count_launch(ctx);
      size_t tb = 0;
      SK_CUDA(cub::DeviceRadixSort::SortPairsDescending(nullptr, tb, ws.chunk_size, ws.chunk_size_sorted, ws.chunk_id, ws.chunk_perm, (int)TC, 0, 32, st));
      SK_TRY(ensure(ctx, &S.sort_tmp, &S.c_sort_tmp, tb));
      SK_CUDA(cub::DeviceRadixSort::SortPairsDescending(S.sort_tmp, tb, ws.chunk_size, ws.chunk_size_sorted, ws.chunk_id, ws.chunk_perm, (int)TC, 0, 32, st));
      // the debug taps run the instantiation production runs, with the score / pointer stores as the only difference
#define DPG(GLV, NEV)                                                                                                   \
  {                                                                                                                    \
    if (taps) SK_TRY((launch_dp_group<true, GLV, NEV>(ctx, g4, TC, prm, ws, dp_minb)));                                \
    else SK_TRY((launch_dp_group<false, GLV, NEV>(ctx, g4, TC, prm, ws, dp_minb)));                                   \
  }
      if (dp_gl == 4) { if (prm.band <= 20) DPG(4, 5) else DPG(4, 6) }
      else { DPG(8, 3) }
#undef DPG
    } else if (nb <= 2) { DP_LAUNCH(2) } else if (nb <= 4) { DP_LAUNCH(4) } else if (nb <= 8) { DP_LAUNCH(8) }
    else if (nb <= 16) { DP_LAUNCH(16) } else { ctx->err = "c too small: chain band > 479 anchors is not supported"; return SK_ERR_PARAM; }
#undef DP_LAUNCH
  }
  SK_LAUNCH(ctx, "select_kernel", (select_kernel<<<B, CT, 0, st>>>(S.d_pairs, prm, ws)));
  return SK_OK;
}

// Copies the intermediate products of every pair of the batch out of the batch arrays: pair i's anchors at pairAbase[i],
// its chunks at pairCbase[i], its intervals at pairIbase[i] (pair_nint[i] of them, sorted order at iv_order + 4 ib + npow2,
// kept flags at iv_kept + ib, both indexed by the pair-local interval index).  dbg[b0 + i] receives pair b0 + i.
static int copy_out_debug(sk_ctx* ctx, const Workspace& ws, const std::vector<PairDesc>& descs, size_t b0, uint32_t B,
                          const std::vector<uint64_t>& abase, const std::vector<uint64_t>& cbase, const std::vector<uint64_t>& ibase,
                          const uint32_t* dbg_counts, const sk_ani_result* host_out, sk_chain_debug* dbg) {
  const uint64_t TA = abase[B], TC = cbase[B], TI = ibase[B];
  std::vector<AnchorRec> anc(TA);
  std::vector<int32_t> score(TA);
  std::vector<uint32_t> ptr(TA), cq(TC), nseeds(TC), nint(B), w(TC), order(4 * TI);
  std::vector<uint64_t> cf(TC + 1);
  std::vector<IntervalKey> iv(TI);
  std::vector<uint8_t> kept(TI), valid(TC);
  std::vector<double> est(TC);
  std::vector<uint32_t> a_total(TC), a_rq0(TC), a_rq1(TC), a_tbcq(TC), a_nint(TC), counts(3 * TC);
  if (TA) {
    SK_CUDA(cudaMemcpy(anc.data(), ws.anc, TA * sizeof(AnchorRec), cudaMemcpyDeviceToHost));
    SK_CUDA(cudaMemcpy(score.data(), ws.score, TA * 4, cudaMemcpyDeviceToHost));
    SK_CUDA(cudaMemcpy(ptr.data(), ws.ptr, TA * 4, cudaMemcpyDeviceToHost));
  }
  if (TC) {
    SK_CUDA(cudaMemcpy(cf.data(), ws.chunk_first, (TC + 1) * 8, cudaMemcpyDeviceToHost));
    SK_CUDA(cudaMemcpy(cq.data(), ws.chunk_qctg, TC * 4, cudaMemcpyDeviceToHost));
    SK_CUDA(cudaMemcpy(nseeds.data(), ws.chunk_nseeds, TC * 4, cudaMemcpyDeviceToHost));
    SK_CUDA(cudaMemcpy(est.data(), ws.chunk_est, TC * 8, cudaMemcpyDeviceToHost));
    SK_CUDA(cudaMemcpy(w.data(), ws.chunk_w, TC * 4, cudaMemcpyDeviceToHost));
    SK_CUDA(cudaMemcpy(valid.data(), ws.chunk_valid, TC, cudaMemcpyDeviceToHost));
    SK_CUDA(cudaMemcpy(a_total.data(), ws.acc_total, TC * 4, cudaMemcpyDeviceToHost));
    SK_CUDA(cudaMemcpy(a_rq0.data(), ws.acc_rq0, TC * 4, cudaMemcpyDeviceToHost));
    SK_CUDA(cudaMemcpy(a_rq1.data(), ws.acc_rq1, TC * 4, cudaMemcpyDeviceToHost));
    SK_CUDA(cudaMemcpy(a_tbcq.data(), ws.acc_tbcq, TC * 4, cudaMemcpyDeviceToHost));
    SK_CUDA(cudaMemcpy(a_nint.data(), ws.acc_nint, TC * 4, cudaMemcpyDeviceToHost));
    SK_CUDA(cudaMemcpy(counts.data(), dbg_counts, TC * 12, cudaMemcpyDeviceToHost));
  }
  SK_CUDA(cudaMemcpy(nint.data(), ws.pair_nint, B * 4, cudaMemcpyDeviceToHost));
  if (TI) {
    // a pair's sorted order ends at 4 ib + npow2 + n < 4 ib + 3 n <= 4 (ib + capacity): inside the batch's 4 TI entries
    SK_CUDA(cudaMemcpy(iv.data(), ws.iv, TI * sizeof(IntervalKey), cudaMemcpyDeviceToHost));
    SK_CUDA(cudaMemcpy(order.data(), ws.iv_order, 4 * TI * 4, cudaMemcpyDeviceToHost));
    SK_CUDA(cudaMemcpy(kept.data(), ws.iv_kept, TI, cudaMemcpyDeviceToHost));
  }
  for (uint32_t i = 0; i < B; i++) {
    sk_chain_debug* d = dbg + b0 + i;
    memset(d, 0, sizeof(*d));
    d->result = host_out[b0 + i];
    d->switched = descs[b0 + i].switched;
    const uint64_t a0 = abase[i], na = abase[i + 1] - a0, c0 = cbase[i], nc = cbase[i + 1] - c0, ib = ibase[i];
    const uint32_t ni = nint[i];
    if (ni > ibase[i + 1] - ib) { ctx->err = "chain debug: a pair has more intervals than its capacity"; return SK_ERR_STATE; }
    d->n_anchors = na; d->n_chunks = nc; d->n_intervals = ni;
    d->anchors = (uint32_t*)calloc(std::max<uint64_t>(na, 1), 20);
    d->score = (int64_t*)calloc(std::max<uint64_t>(na, 1), 8);
    d->pointer = (uint32_t*)calloc(std::max<uint64_t>(na, 1), 4);
    d->chunk_first = (uint32_t*)calloc(nc + 1, 4);
    d->chunk_nseeds = (uint32_t*)calloc(std::max<uint64_t>(nc, 1), 4);
    d->intervals = (int64_t*)calloc(std::max<uint32_t>(ni, 1), 11 * 8);
    d->chunk_stats = (uint32_t*)calloc(std::max<uint64_t>(nc, 1), 9 * 4);
    if (!d->anchors || !d->score || !d->pointer || !d->chunk_first || !d->chunk_nseeds || !d->intervals || !d->chunk_stats) {
      ctx->err = "chain debug: out of host memory"; return SK_ERR_STATE;
    }
    for (uint64_t c = 0; c < nc; c++) {
      // chunk_first is batch-global; the pair's last chunk ends where the next pair's anchors (or the sentinel) begin
      const uint64_t x0 = cf[c0 + c] - a0, x1 = cf[c0 + c + 1] - a0;
      if (x0 > x1 || x1 > na) { ctx->err = "chain debug: chunk outside its pair's anchors"; return SK_ERR_STATE; }
      d->chunk_first[c] = (uint32_t)x0; d->chunk_nseeds[c] = nseeds[c0 + c];
      const uint64_t g = c0 + c;
      const uint32_t st[9] = {a_total[g], a_rq0[g], a_rq1[g], a_tbcq[g], a_nint[g], nseeds[g], counts[3 * g], counts[3 * g + 1],
                              counts[3 * g + 2]};
      memcpy(d->chunk_stats + 9 * c, st, sizeof(st));
      for (uint64_t x = x0; x < x1; x++) {
        const AnchorRec& a = anc[a0 + x];
        uint32_t* o = d->anchors + 5 * x;
        o[0] = cq[c0 + c]; o[1] = a.qpos; o[2] = a.rc >> 1; o[3] = a.rpos; o[4] = a.rc & 1u;
        d->score[x] = score[a0 + x]; d->pointer[x] = ptr[a0 + x];
      }
    }
    d->chunk_first[nc] = (uint32_t)na;
    uint32_t npow2 = 1;
    while (npow2 < ni) npow2 <<= 1;
    for (uint32_t j = 0; j < ni; j++) {
      const uint32_t oj = order[4 * ib + npow2 + j];
      if (oj >= ni) { ctx->err = "chain debug: interval order out of range"; return SK_ERR_STATE; }
      const IntervalKey& x = iv[ib + oj];
      int64_t* o = d->intervals + 11 * j;
      o[0] = iv_score(x); o[1] = iv_num_anchors(x); o[2] = iv_q0(x); o[3] = iv_q1(x); o[4] = iv_r0(x); o[5] = iv_r1(x);
      o[6] = iv_rctg(x); o[7] = iv_qctg(x); o[8] = iv_chunk(x); o[9] = iv_rev(x); o[10] = kept[ib + oj];
    }
    std::vector<std::pair<double, uint64_t>> es;
    for (uint64_t c = c0; c < c0 + nc; c++) if (valid[c]) es.push_back({est[c], w[c]});
    std::sort(es.begin(), es.end());
    d->n_ests = es.size();
    d->est = (double*)calloc(std::max<size_t>(es.size(), 1), 8);
    d->weight = (uint64_t*)calloc(std::max<size_t>(es.size(), 1), 8);
    if (!d->est || !d->weight) { ctx->err = "chain debug: out of host memory"; return SK_ERR_STATE; }
    for (size_t j = 0; j < es.size(); j++) { d->est[j] = es[j].first; d->weight[j] = es[j].second; }
  }
  return SK_OK;
}

// Runs one batch (pairs [b0, b1) of `descs`); results -> host_out[b0..b1).  If dbg != nullptr (one entry per pair of the
// whole list) the intermediate products of the batch's pairs are copied out as well.
static int run_batch(sk_ctx* ctx, ChainScratch& S, const sk_sketch_set* refs, const sk_sketch_set* qs, const std::vector<PairDesc>& descs,
                     size_t b0, size_t b1, uint64_t total_rec, uint64_t total_chunks, const std::vector<uint32_t>& tile_off, const ChainParams& prm, const SetView& v0, const SetView& v1,
                     sk_ani_result* host_out, sk_chain_debug* dbg, MapOut* mo) {
  cudaStream_t st = ctx->stream;
  const uint32_t B = (uint32_t)(b1 - b0);
  Workspace& ws = S.ws;
  const size_t NR = std::max<uint64_t>(total_rec, 1);
#define ENS(field, capf, n) SK_TRY(ensure(ctx, &ws.field, &S.capf, n))
  const size_t NS = std::max<uint64_t>(total_chunks, 1);
  const size_t NT = std::max<uint32_t>(tile_off[B], 1);
  ENS(hit, c_hit, NR); ENS(tile_hits, c_tile_hits, NT); ENS(rec_cnt, c_rec_cnt, NT * (TILE / 32)); ENS(tile_off, c_tile_off, B + 1);
  ENS(stg_first, c_stg_first, NS); ENS(stg_qctg, c_stg_qctg, NS); ENS(stg_lo, c_stg_lo, NS); ENS(stg_hi, c_stg_hi, NS);
  ENS(pairA, c_pairA, B); ENS(pairC, c_pairC, B); ENS(pairAbase, c_pairAbase, B + 1); ENS(pairCbase, c_pairCbase, B + 1);
  ENS(pairIbase, c_pairIbase, B + 1); ENS(pair_nint, c_pair_nint, B); ENS(pair_sumlen, c_pair_sumlen, B); ENS(pair_nchains, c_pair_nchains, B);
  ENS(pair_tqb_ns, c_pair_tqb, B);
  SK_TRY(ensure(ctx, &S.d_pairs, &S.c_pairs, B));
  SK_TRY(ensure(ctx, &S.d_out, &S.c_out, B));
  SK_CUDA(h2d_small(ctx, S.d_pairs, descs.data() + b0, B * sizeof(PairDesc)));
  SK_CUDA(cudaMemsetAsync(ws.pair_nint, 0, B * 4, st));
  SK_CUDA(cudaMemsetAsync(ws.pair_sumlen, 0, B * 4, st));
  SK_CUDA(cudaMemsetAsync(ws.pair_nchains, 0, B * 4, st));
  SK_CUDA(cudaMemsetAsync(ws.pair_tqb_ns, 0, B * 4, st));
  SK_CUDA(cudaMemsetAsync(ws.pairA, 0, B * 4, st));
  SK_CUDA(h2d_small(ctx, ws.tile_off, tile_off.data(), (B + 1) * 4));

  const uint32_t n_tiles = tile_off[B];
  if (n_tiles > 0) {
    // small ref-role genomes (k-mer table <= 16 KB): TMA-stage the table in shared memory when they dominate the batch
    size_t n_small = 0;
    for (size_t i = b0; i < b1; i++) {
      const PairDesc& d = descs[i];
      if (!d.valid) continue;
      const sk_sketch_set* rs_ = d.rset ? qs : refs;
      if (!rs_->ht_off.empty()) { const uint64_t cap = rs_->ht_off[d.rg + 1] - rs_->ht_off[d.rg]; if (cap && cap <= PROBE_STAGE_ENTRIES) n_small++; }
    }
    const bool staged = (getenv("SK_PROBE_TMA") ? atoi(getenv("SK_PROBE_TMA")) != 0 : true) && 2 * n_small >= (size_t)B;
    if (staged) SK_LAUNCH(ctx, "probe_kernel", (probe_kernel<true, PROBE_MINB><<<n_tiles, CT, 0, st>>>(S.d_pairs, B, v0, v1, S.d_m0, S.d_m1, prm, ws)));
    else SK_LAUNCH(ctx, "probe_kernel", (probe_kernel<false, PROBE_MINB><<<n_tiles, CT, 0, st>>>(S.d_pairs, B, v0, v1, S.d_m0, S.d_m1, prm, ws)));
  }
  std::vector<uint32_t> hA(B), hC(B);
  SK_CUDA(cudaMemcpyAsync(hA.data(), ws.pairA, B * 4, cudaMemcpyDeviceToHost, st));
  SK_CUDA(cudaStreamSynchronize(st));
  SK_CUDA(cudaGetLastError());
  std::vector<uint64_t> abase(B + 1, 0), cbase(B + 1, 0), ibase(B + 1, 0);
  for (uint32_t i = 0; i < B; i++) {
    abase[i + 1] = abase[i] + hA[i];
    ibase[i + 1] = ibase[i] + hA[i] / 3;   // every chain interval owns >= 3 distinct anchors
  }
  const uint64_t TA = abase[B], TI = ibase[B];
  SK_CUDA(h2d_small(ctx, ws.pairAbase, abase.data(), (B + 1) * 8));
  SK_CUDA(h2d_small(ctx, ws.pairIbase, ibase.data(), (B + 1) * 8));
  const size_t NA = std::max<uint64_t>(TA, 1), NI = std::max<uint64_t>(TI, 1);
  ENS(anc, c_anc, NA);
  SK_CUDA(cudaFuncSetAttribute(chunk_anchor_kernel<CHUNK_ANCHOR_MINB>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                               (int)sizeof(ChunkAnchorSmem)));
  SK_LAUNCH(ctx, "chunk_anchor_kernel", (chunk_anchor_kernel<CHUNK_ANCHOR_MINB><<<B, CT, sizeof(ChunkAnchorSmem), st>>>(S.d_pairs, v0, v1, S.d_m0, S.d_m1, ws)));
  SK_CUDA(cudaMemcpyAsync(hC.data(), ws.pairC, B * 4, cudaMemcpyDeviceToHost, st));
  SK_CUDA(cudaStreamSynchronize(st));
  SK_CUDA(cudaGetLastError());
  for (uint32_t i = 0; i < B; i++) {
    if (hC[i] > descs[b0 + i].max_chunks) { ctx->err = "chain: a pair has more chunks than its contig-length bound"; return SK_ERR_STATE; }
    cbase[i + 1] = cbase[i] + hC[i];
  }
  const uint64_t TC = cbase[B];
  SK_CUDA(h2d_small(ctx, ws.pairCbase, cbase.data(), (B + 1) * 8));
  const size_t NCH = std::max<uint64_t>(TC, 1);
  ENS(score, c_score, dbg ? NA : 1); ENS(ptr, c_ptr, dbg ? NA : 1); ENS(rootkey, c_rootkey, NA); ENS(depth, c_depth, NA);
  ENS(chunk_first, c_chunk_first, NCH + 1); ENS(chunk_pair, c_chunk_pair, NCH); ENS(chunk_qctg, c_chunk_qctg, NCH);
  ENS(chunk_lo, c_chunk_lo, NCH); ENS(chunk_hi, c_chunk_hi, NCH); ENS(acc_total, c_acc_total, NCH); ENS(acc_rq0, c_acc_rq0, NCH);
  ENS(acc_rq1, c_acc_rq1, NCH); ENS(acc_tbcq, c_acc_tbcq, NCH); ENS(acc_nint, c_acc_nint, NCH); ENS(chunk_head, c_chunk_head, NCH);
  ENS(chunk_est, c_chunk_est, NCH); ENS(chunk_w, c_chunk_w, NCH); ENS(chunk_valid, c_chunk_valid, NCH); ENS(chunk_nseeds, c_chunk_nseeds, NCH);
  ENS(iv, c_iv, NI); ENS(iv_keys, c_iv_keys, 2 * NI + 8); ENS(iv_order, c_iv_order, 4 * NI + 8); ENS(iv_kept, c_iv_kept, NI); ENS(iv_next, c_iv_next, NI); ENS(acc_list, c_acc_list, NI);
  ENS(est_sorted, c_est_sorted, 4 * NCH + 8); ENS(w_sorted, c_w_sorted, 4 * NCH + 8);
#undef ENS
  if (dbg) SK_TRY(ensure(ctx, &S.dbg_counts, &S.c_dbg_counts, 3 * NCH));
  uint32_t* const dbg_counts = dbg ? S.dbg_counts : nullptr;
  if (TC > 0) {
    SK_CUDA(h2d_small(ctx, ws.chunk_first + TC, &TA, 8));
    SK_LAUNCH(ctx, "chunk_compact_kernel", (chunk_compact_kernel<<<B, CT, 0, st>>>(S.d_pairs, ws)));
    init_chunk_acc_kernel<<<(uint32_t)((TC + 255) / 256), 256, 0, st>>>(TC, ws); count_launch(ctx);
    SK_TRY(launch_dp_select(ctx, S, B, TC, prm, true, dbg != nullptr));
    SK_LAUNCH(ctx, "chunkstat_kernel", (chunkstat_kernel<<<(uint32_t)((TC + CS_WARPS * CS_PER_WARP - 1) / (CS_WARPS * CS_PER_WARP)), CS_WARPS * 32, 0, st>>>(TC, S.d_pairs, v0, v1, S.d_m0, S.d_m1, prm, ws, dbg_counts)));
  }
  std::vector<uint64_t> hmap(mo ? B + 1 : 0);
  if (mo) {
    // every pair's kept intervals (pair_nchains of them, acc_list) as sorted records, offsets and records copied out below
    SK_TRY(ensure(ctx, &S.map_base, &S.c_map_base, B + 1));
    SK_TRY(ensure(ctx, &S.map_out, &S.c_map_out, NI)); SK_TRY(ensure(ctx, &S.map_stage, &S.c_map_stage, NI));
    SK_TRY(ensure(ctx, &S.map_idx, &S.c_map_idx, 2 * NI));
    SK_LAUNCH(ctx, "mapping_scan_kernel", (mapping_scan_kernel<<<1, MAP_SCAN_T, 0, st>>>(B, ws.pair_nchains, S.map_base)));
    SK_LAUNCH(ctx, "mapping_emit_kernel", (mapping_emit_kernel<<<B, CT, 0, st>>>(S.d_pairs, ws, S.map_base, S.map_stage, S.map_idx, S.map_out)));
    SK_CUDA(cudaMemcpyAsync(hmap.data(), S.map_base, (B + 1) * 8, cudaMemcpyDeviceToHost, st));
  }
  // test hook: SK_FINAL_FORCE_REDO=1 takes the sequential bootstrap redo for every pair, as if some draw had been rejected
  const char* fr = getenv("SK_FINAL_FORCE_REDO");
  const int force_redo = (fr && atoi(fr) != 0) ? 1 : 0;
  SK_LAUNCH(ctx, "final_kernel", (final_kernel<<<B, FT, 0, st>>>(S.d_pairs, S.d_m0, S.d_m1, prm, ws, S.d_out, force_redo)));
  SK_CUDA(cudaMemcpyAsync(host_out + b0, S.d_out, B * sizeof(sk_ani_result), cudaMemcpyDeviceToHost, st));
  SK_CUDA(cudaStreamSynchronize(st));
  SK_CUDA(cudaGetLastError());

  if (mo) {
    const uint64_t n = hmap[B];
    if (n > TI) { ctx->err = "chain mappings: more kept intervals than the batch's interval capacity"; return SK_ERR_STATE; }
    if (mo->n + n > mo->cap) {
      const size_t cap = std::max<size_t>(mo->n + n, 2 * mo->cap);
      sk_mapping* r = (sk_mapping*)realloc(mo->recs, std::max<size_t>(cap, 1) * sizeof(sk_mapping));
      if (!r) { ctx->err = "chain mappings: out of host memory"; return SK_ERR_NOMEM; }
      mo->recs = r; mo->cap = cap;
    }
    if (n) {
      if (n > S.c_h_map) {   // grow-only pinned staging: the copy runs at full PCIe rate
        if (S.h_map) SK_CUDA(cudaFreeHost(S.h_map));
        S.h_map = nullptr; S.c_h_map = 0;
        const size_t c = n + n / 4;
        SK_CUDA(cudaMallocHost((void**)&S.h_map, c * sizeof(sk_mapping)));
        S.c_h_map = c;
      }
      SK_CUDA(cudaMemcpyAsync(S.h_map, S.map_out, n * sizeof(sk_mapping), cudaMemcpyDeviceToHost, st));
      SK_CUDA(cudaStreamSynchronize(st));
      memcpy(mo->recs + mo->n, S.h_map, n * sizeof(sk_mapping));
      mo->n += n;
    }
    for (uint32_t i = 0; i < B; i++) mo->count[b0 + i] = hmap[i + 1] - hmap[i];
  }
  if (dbg) SK_TRY(copy_out_debug(ctx, ws, descs, b0, B, abase, cbase, ibase, dbg_counts, host_out, dbg));
  return SK_OK;
}

static ChainScratch& chain_scratch(sk_ctx* ctx) {
  if (!ctx->chain_scratch) {
    ctx->chain_scratch = new ChainScratch();
    ctx->chain_scratch_free = [](void* p) { ((ChainScratch*)p)->free_all(); delete (ChainScratch*)p; };
  }
  return *(ChainScratch*)ctx->chain_scratch;   // grow-only device buffers, reused by every call on this context
}

// Test entries: the workspace of B pairs filled from host lists the way chunk_anchor_kernel / chunk_compact_kernel (anchors,
// chunk descriptors, pair bases; h_anc non-empty) or the DP (intervals and their counts; h_iv non-empty) leave it, then
// launch_dp_select and copy_out_debug as a debug run of run_batch.  cbase / abase / ibase: per-pair exclusive prefixes (B + 1).
static int debug_dp_select(sk_ctx* ctx, uint32_t c, uint32_t k, const uint32_t* switched, const std::vector<uint64_t>& cbase,
                           const std::vector<uint64_t>& abase, const std::vector<uint64_t>& ibase, const std::vector<AnchorRec>& h_anc,
                           const std::vector<uint64_t>& h_first, const std::vector<uint32_t>& h_qctg,
                           const std::vector<IntervalKey>& h_iv, const std::vector<uint32_t>& h_nint, bool dp, sk_chain_debug* out,
                           uint32_t* pair_sums) {
  SK_CUDA(cudaSetDevice(ctx->device));
  cudaStream_t st = ctx->stream;
  const uint32_t B = (uint32_t)(cbase.size() - 1);
  ChainParams prm{};
  prm.c = c; prm.k = k; prm.band = BP_CHAIN_BAND / c; prm.model = -1;
  if (prm.band / 32 + 2 > 16) { ctx->err = "c too small: chain band > 479 anchors is not supported"; return SK_ERR_PARAM; }
  ChainScratch& S = chain_scratch(ctx);
  Workspace& ws = S.ws;
  const uint64_t TA = abase[B], TC = cbase[B], TI = ibase[B];
  const size_t NA = std::max<uint64_t>(TA, 1), NCH = std::max<uint64_t>(TC, 1), NI = std::max<uint64_t>(TI, 1);
#define ENS(field, capf, n) SK_TRY(ensure(ctx, &ws.field, &S.capf, n))
  ENS(pairCbase, c_pairCbase, B + 1); ENS(pairIbase, c_pairIbase, B + 1); ENS(pair_nint, c_pair_nint, B);
  ENS(pair_sumlen, c_pair_sumlen, B); ENS(pair_nchains, c_pair_nchains, B);
  ENS(anc, c_anc, NA); ENS(score, c_score, NA); ENS(ptr, c_ptr, NA); ENS(rootkey, c_rootkey, NA); ENS(depth, c_depth, NA);
  ENS(chunk_first, c_chunk_first, NCH + 1); ENS(chunk_pair, c_chunk_pair, NCH); ENS(chunk_qctg, c_chunk_qctg, NCH);
  ENS(acc_total, c_acc_total, NCH); ENS(acc_rq0, c_acc_rq0, NCH); ENS(acc_rq1, c_acc_rq1, NCH); ENS(acc_tbcq, c_acc_tbcq, NCH);
  ENS(acc_nint, c_acc_nint, NCH); ENS(chunk_head, c_chunk_head, NCH); ENS(chunk_est, c_chunk_est, NCH); ENS(chunk_w, c_chunk_w, NCH);
  ENS(chunk_valid, c_chunk_valid, NCH); ENS(chunk_nseeds, c_chunk_nseeds, NCH);
  ENS(iv, c_iv, NI); ENS(iv_keys, c_iv_keys, 2 * NI + 8); ENS(iv_order, c_iv_order, 4 * NI + 8); ENS(iv_kept, c_iv_kept, NI);
  ENS(iv_next, c_iv_next, NI); ENS(acc_list, c_acc_list, NI);
#undef ENS
  SK_TRY(ensure(ctx, &S.dbg_counts, &S.c_dbg_counts, 3 * NCH));
  SK_TRY(ensure(ctx, &S.d_pairs, &S.c_pairs, B));
  std::vector<PairDesc> descs(B);
  std::vector<uint32_t> h_pair(TC);
  for (uint32_t p = 0; p < B; p++) {
    PairDesc& d = descs[p];
    memset(&d, 0, sizeof(d));
    d.switched = switched[p] ? 1 : 0; d.valid = 1;
    for (uint64_t i = cbase[p]; i < cbase[p + 1]; i++) h_pair[i] = p;
  }
  SK_CUDA(cudaMemcpyAsync(S.d_pairs, descs.data(), B * sizeof(PairDesc), cudaMemcpyHostToDevice, st));
  SK_CUDA(cudaMemcpyAsync(ws.pairCbase, cbase.data(), (B + 1) * 8, cudaMemcpyHostToDevice, st));
  SK_CUDA(cudaMemcpyAsync(ws.pairIbase, ibase.data(), (B + 1) * 8, cudaMemcpyHostToDevice, st));
  SK_CUDA(cudaMemsetAsync(ws.pair_sumlen, 0, B * 4, st));
  SK_CUDA(cudaMemsetAsync(ws.pair_nchains, 0, B * 4, st));
  if (dp) SK_CUDA(cudaMemsetAsync(ws.pair_nint, 0, B * 4, st));
  else SK_CUDA(cudaMemcpyAsync(ws.pair_nint, h_nint.data(), B * 4, cudaMemcpyHostToDevice, st));
  if (TA) {
    SK_CUDA(cudaMemcpyAsync(ws.anc, h_anc.data(), TA * sizeof(AnchorRec), cudaMemcpyHostToDevice, st));
    SK_CUDA(cudaMemsetAsync(ws.score, 0, TA * 4, st));
    SK_CUDA(cudaMemsetAsync(ws.ptr, 0, TA * 4, st));
  }
  SK_CUDA(cudaMemcpyAsync(ws.chunk_first, h_first.data(), (TC + 1) * 8, cudaMemcpyHostToDevice, st));
  if (TC) {
    SK_CUDA(cudaMemcpyAsync(ws.chunk_pair, h_pair.data(), TC * 4, cudaMemcpyHostToDevice, st));
    SK_CUDA(cudaMemcpyAsync(ws.chunk_qctg, h_qctg.data(), TC * 4, cudaMemcpyHostToDevice, st));
    // no seeds here: chunkstat_kernel's outputs, which copy_out_debug also reads, are zero
    SK_CUDA(cudaMemsetAsync(ws.chunk_nseeds, 0, TC * 4, st));
    SK_CUDA(cudaMemsetAsync(ws.chunk_valid, 0, TC, st));
    SK_CUDA(cudaMemsetAsync(S.dbg_counts, 0, TC * 12, st));
  }
  if (TI && !dp) SK_CUDA(cudaMemcpyAsync(ws.iv, h_iv.data(), TI * sizeof(IntervalKey), cudaMemcpyHostToDevice, st));
  if (TC) {
    init_chunk_acc_kernel<<<(uint32_t)((TC + 255) / 256), 256, 0, st>>>(TC, ws); count_launch(ctx);
    SK_TRY(launch_dp_select(ctx, S, B, TC, prm, dp, true));
  }
  std::vector<sk_ani_result> res(B);
  memset(res.data(), 0, B * sizeof(sk_ani_result));
  std::vector<uint32_t> sl(B), nc(B);
  SK_CUDA(cudaMemcpyAsync(sl.data(), ws.pair_sumlen, B * 4, cudaMemcpyDeviceToHost, st));
  SK_CUDA(cudaMemcpyAsync(nc.data(), ws.pair_nchains, B * 4, cudaMemcpyDeviceToHost, st));
  SK_CUDA(cudaStreamSynchronize(st));
  SK_CUDA(cudaGetLastError());
  for (uint32_t p = 0; p < B; p++) { pair_sums[2 * p] = sl[p]; pair_sums[2 * p + 1] = nc[p]; }
  return copy_out_debug(ctx, ws, descs, 0, B, abase, cbase, ibase, S.dbg_counts, res.data(), out);
}

static int chain_impl(sk_ctx* ctx, const sk_sketch_set* refs, const sk_sketch_set* qs, const uint64_t* pairs, uint64_t n_pairs,
                      const sk_map_params* mp, sk_ani_result* out, sk_chain_debug* dbg, MapOut* mo) {
  SK_CUDA(cudaSetDevice(ctx->device));
  if (refs->sp.c != qs->sp.c || refs->sp.k != qs->sp.k) { ctx->err = "ref/query sketch parameters differ"; return SK_ERR_PARAM; }
  if (n_pairs == 0) return SK_OK;
  SK_TRY(upload_tables(ctx));
  ChainParams prm;
  prm.c = refs->sp.c; prm.k = refs->sp.k;
  prm.band = BP_CHAIN_BAND / refs->sp.c;                       // index_chain_band (src/chain.rs:111-112)
  prm.ushift = 2 * refs->sp.k > UBUCKET_BITS ? 2 * refs->sp.k - UBUCKET_BITS : 0;
  prm.robust = mp->robust; prm.median = mp->median;
  double fcc = mp->min_aligned_frac;
  if (fcc < 0.) fcc = 15.0 / 100.;                              // src/chain.rs:101-107
  prm.frac_cover_cutoff = fcc;
  prm.both_frac_cover_cutoff = mp->both_min_aligned_frac;
  prm.model = -1;
  if (mp->learned_ani) {                                        // regression::get_model (src/regression.rs:12-28)
    long d125 = std::labs((long)refs->sp.c - 125), d200 = std::labs((long)refs->sp.c - 200);
    prm.model = d125 < d200 ? 0 : 1;
  }
  // dp_warp_kernel holds at most 16 register sets of 32 anchors (band / 32 + 2 <= 16): refused before anything is launched
  if (prm.band / 32 + 2 > 16) { ctx->err = "c too small: chain band > 479 anchors is not supported"; return SK_ERR_PARAM; }
  const bool same = (refs == qs);
  ChainScratch& S = chain_scratch(ctx);
  std::vector<GenomeMeta> m0, m1;
  build_meta(refs, m0);
  build_meta(qs, m1);
  SK_TRY(ensure(ctx, &S.d_m0, &S.c_m0, m0.size()));
  SK_TRY(ensure(ctx, &S.d_m1, &S.c_m1, m1.size()));
  SK_CUDA(h2d_small(ctx, S.d_m0, m0.data(), m0.size() * sizeof(GenomeMeta)));
  SK_CUDA(h2d_small(ctx, S.d_m1, m1.data(), m1.size() * sizeof(GenomeMeta)));
  const SetView v0 = view_of(refs), v1 = view_of(qs);
  // pair descriptors
  std::vector<PairDesc> descs(n_pairs);
  for (uint64_t i = 0; i < n_pairs; i++) {
    uint32_t r = (uint32_t)(pairs[i] >> 32), q = (uint32_t)pairs[i];
    if (r >= refs->G || q >= qs->G) { ctx->err = "pair index out of range"; return SK_ERR_PARAM; }
    PairDesc& d = descs[i];
    d.ref_idx = r; d.query_idx = q; d.rec_off = 0; d.chunk_off = 0; d.max_chunks = 0; d.pad = 0;
    bool empty = (m0[r].n_ctg == 0 || m1[q].n_ctg == 0);      // src/chain.rs:618-620
    d.valid = empty ? 0 : 1;
    bool sw = empty ? true : pair_switched(refs, r, qs, q, same);
    d.switched = sw ? 1 : 0;
    if (sw) { d.qset = 0; d.qg = r; d.rset = 1; d.rg = q; }    // iterate + chunk the ref sketch, probe the query sketch
    else { d.qset = 1; d.qg = q; d.rset = 0; d.rg = r; }
  }
  // batches bounded by the per-record workspace
  const uint64_t REC_CAP = 128ull << 20;
  std::vector<uint32_t> tile_off;   // exclusive prefix of probe tiles per pair of the batch
  size_t b0 = 0;
  while (b0 < n_pairs) {
    size_t b1 = b0;
    uint64_t rec = 0, chunks = 0;
    tile_off.assign(1, 0);
    while (b1 < n_pairs && b1 - b0 < 65535) {
      PairDesc& d = descs[b1];
      const GenomeMeta* qm = d.valid ? &(d.qset ? m1 : m0)[d.qg] : nullptr;
      const uint64_t nr = qm ? qm->n_rec : 0;
      if (b1 > b0 && rec + nr > REC_CAP) break;
      d.rec_off = rec;
      d.chunk_off = chunks;
      d.max_chunks = qm ? qm->max_chunks : 0;
      rec += nr; chunks += d.max_chunks;
      tile_off.push_back(tile_off.back() + (uint32_t)((nr + TILE - 1) / TILE));
      b1++;
    }
    SK_TRY(run_batch(ctx, S, refs, qs, descs, b0, b1, rec, chunks, tile_off, prm, v0, v1, out, dbg, mo));
    b0 = b1;
  }
  return SK_OK;
}

}  // namespace sk

extern "C" {

int sk_chain_pairs(sk_ctx* ctx, const sk_sketch_set* refs, const sk_sketch_set* queries, const uint64_t* pairs, uint64_t n_pairs,
                   const sk_map_params* mp, sk_ani_result* out) {
  if (!ctx || !refs || !queries || !mp || (n_pairs && (!pairs || !out))) return SK_ERR_PARAM;
  return sk::chain_impl(ctx, refs, queries, pairs, n_pairs, mp, out, nullptr, nullptr);
}

int sk_chain_pairs_mappings(sk_ctx* ctx, const sk_sketch_set* refs, const sk_sketch_set* queries, const uint64_t* pairs,
                            uint64_t n_pairs, const sk_map_params* mp, sk_ani_result* out, uint64_t* map_off, sk_mapping** maps) {
  if (!ctx || !refs || !queries || !mp || !map_off || !maps || (n_pairs && (!pairs || !out))) return SK_ERR_PARAM;
  *maps = nullptr;
  sk::MapOut mo;
  mo.count.assign(n_pairs, 0);
  SK_TRY(sk::chain_impl(ctx, refs, queries, pairs, n_pairs, mp, out, nullptr, &mo));
  map_off[0] = 0;
  for (uint64_t i = 0; i < n_pairs; i++) map_off[i + 1] = map_off[i] + mo.count[i];
  if (!mo.recs) mo.recs = (sk_mapping*)malloc(sizeof(sk_mapping));
  if (!mo.recs) { ctx->err = "chain mappings: out of host memory"; return SK_ERR_NOMEM; }
  *maps = mo.recs;
  mo.recs = nullptr;
  return SK_OK;
}

void sk_chain_debug_free(sk_chain_debug* d) {
  if (!d) return;
  free(d->anchors); free(d->chunk_first); free(d->chunk_nseeds); free(d->score); free(d->pointer); free(d->intervals);
  free(d->est); free(d->weight); free(d->chunk_stats);
  memset(d, 0, sizeof(*d));
}

int sk_debug_chunk_estimate(sk_ctx* ctx, uint64_t n, const uint32_t* inputs, uint32_t c, uint32_t k, double* est, uint32_t* weight,
                            uint32_t* valid) {
  if (!ctx || (n && (!inputs || !est || !weight || !valid)) || k == 0) return SK_ERR_PARAM;
  if (n == 0) return SK_OK;
  SK_CUDA(cudaSetDevice(ctx->device));
  cudaStream_t st = ctx->stream;
  uint32_t *d_in = nullptr, *d_w = nullptr, *d_v = nullptr;
  double* d_e = nullptr;
  int rc = SK_OK;
  cudaError_t e = cudaMalloc(&d_in, n * 32);
  if (e == cudaSuccess) e = cudaMalloc(&d_e, n * 8);
  if (e == cudaSuccess) e = cudaMalloc(&d_w, n * 4);
  if (e == cudaSuccess) e = cudaMalloc(&d_v, n * 4);
  if (e == cudaSuccess) e = cudaMemcpyAsync(d_in, inputs, n * 32, cudaMemcpyHostToDevice, st);
  if (e == cudaSuccess) {
    sk::debug_chunk_estimate_kernel<<<(uint32_t)((n + 255) / 256), 256, 0, st>>>(n, d_in, c, k, d_e, d_w, d_v);
    sk::count_launch(ctx);
    e = cudaGetLastError();
  }
  if (e == cudaSuccess) e = cudaMemcpyAsync(est, d_e, n * 8, cudaMemcpyDeviceToHost, st);
  if (e == cudaSuccess) e = cudaMemcpyAsync(weight, d_w, n * 4, cudaMemcpyDeviceToHost, st);
  if (e == cudaSuccess) e = cudaMemcpyAsync(valid, d_v, n * 4, cudaMemcpyDeviceToHost, st);
  if (e == cudaSuccess) e = cudaStreamSynchronize(st);
  if (e != cudaSuccess) { ctx->err = cudaGetErrorString(e); rc = SK_ERR_CUDA; }
  cudaFree(d_in); cudaFree(d_e); cudaFree(d_w); cudaFree(d_v);
  return rc;
}

int sk_debug_chain_anchors(sk_ctx* ctx, uint32_t c, uint32_t k, uint64_t n_pairs, const uint64_t* pair_chunk_off,
                           const uint64_t* chunk_anchor_off, const uint32_t* anchors, const uint32_t* switched, sk_chain_debug* out,
                           uint32_t* pair_sums) {
  if (!ctx || c == 0 || (n_pairs && (!pair_chunk_off || !chunk_anchor_off || !switched || !out || !pair_sums))) return SK_ERR_PARAM;
  if (n_pairs == 0) return SK_OK;
  if (n_pairs > 65535) { ctx->err = "debug chain: at most 65535 pairs"; return SK_ERR_PARAM; }
  memset(out, 0, n_pairs * sizeof(*out));
  const uint64_t TC = pair_chunk_off[n_pairs], TA = chunk_anchor_off[TC];
  if (pair_chunk_off[0] != 0 || chunk_anchor_off[0] != 0 || (TA && !anchors)) return SK_ERR_PARAM;
  std::vector<uint64_t> cbase(n_pairs + 1), abase(n_pairs + 1, 0), ibase(n_pairs + 1, 0), first(TC + 1);
  std::vector<uint32_t> qctg(TC);
  std::vector<sk::AnchorRec> anc(TA);
  for (uint64_t p = 0; p <= n_pairs; p++) {
    cbase[p] = pair_chunk_off[p];
    if (p && cbase[p] < cbase[p - 1]) { ctx->err = "debug chain: pair chunk offsets decrease"; return SK_ERR_PARAM; }
  }
  for (uint64_t p = 0; p < n_pairs; p++) {
    for (uint64_t ch = cbase[p]; ch < cbase[p + 1]; ch++) {
      const uint64_t a0 = chunk_anchor_off[ch], a1 = chunk_anchor_off[ch + 1];
      if (a1 <= a0) { ctx->err = "debug chain: every chunk holds at least one anchor"; return SK_ERR_PARAM; }
      first[ch] = a0;
      qctg[ch] = anchors[5 * a0];
      for (uint64_t i = a0; i < a1; i++) {
        const uint32_t* x = anchors + 5 * i;
        // types.rs:135-138 (contig index < 2^30: the DP's unfilled-set sentinels are no contig) and the sketch-time position bound
        if (x[0] != qctg[ch]) { ctx->err = "debug chain: a chunk holds one query contig"; return SK_ERR_PARAM; }
        if (x[2] >= (1u << 30) || x[4] > 1u) { ctx->err = "debug chain: ref contig >= 2^30 or reverse flag > 1"; return SK_ERR_PARAM; }
        if (x[1] >= 0xFFFF0000u || x[3] >= 0xFFFF0000u) { ctx->err = "debug chain: position >= 2^32 - 65536"; return SK_ERR_PARAM; }
        if (i > a0) {   // the order chunk_anchor_kernel emits: (query_pos, ref_contig, ref_pos, reverse)
          const uint32_t* y = x - 5;
          const bool sorted = y[1] != x[1] ? y[1] < x[1] : y[2] != x[2] ? y[2] < x[2] : y[3] != x[3] ? y[3] < x[3] : y[4] <= x[4];
          if (!sorted) { ctx->err = "debug chain: the anchors of a chunk are not sorted by (qpos, rctg, rpos, rev)"; return SK_ERR_PARAM; }
        }
        anc[i].qpos = x[1]; anc[i].rpos = x[3]; anc[i].rc = (x[2] << 1) | x[4];
      }
    }
    abase[p + 1] = chunk_anchor_off[cbase[p + 1]];
    ibase[p + 1] = ibase[p] + (abase[p + 1] - abase[p]) / 3;   // run_batch's interval capacity
  }
  first[TC] = TA;
  const int rc = sk::debug_dp_select(ctx, c, k, switched, cbase, abase, ibase, anc, first, qctg, {}, {}, true, out, pair_sums);
  if (rc != SK_OK) for (uint64_t i = 0; i < n_pairs; i++) sk_chain_debug_free(out + i);
  return rc;
}

int sk_debug_select_intervals(sk_ctx* ctx, uint32_t c, uint32_t k, uint64_t n_pairs, const uint64_t* pair_iv_off,
                              const int64_t* intervals, const uint32_t* pair_chunks, const uint32_t* switched, sk_chain_debug* out,
                              uint32_t* pair_sums) {
  if (!ctx || c == 0 || (n_pairs && (!pair_iv_off || !pair_chunks || !switched || !out || !pair_sums))) return SK_ERR_PARAM;
  if (n_pairs == 0) return SK_OK;
  if (n_pairs > 65535) { ctx->err = "debug select: at most 65535 pairs"; return SK_ERR_PARAM; }
  memset(out, 0, n_pairs * sizeof(*out));
  const uint64_t TI = pair_iv_off[n_pairs];
  if (pair_iv_off[0] != 0 || (TI && !intervals)) return SK_ERR_PARAM;
  std::vector<uint64_t> cbase(n_pairs + 1, 0), abase(n_pairs + 1, 0), ibase(n_pairs + 1);
  std::vector<uint32_t> nint(n_pairs);
  std::vector<sk::IntervalKey> iv(TI);
  for (uint64_t p = 0; p < n_pairs; p++) {
    cbase[p + 1] = cbase[p] + pair_chunks[p];
    ibase[p] = pair_iv_off[p];
    if (pair_iv_off[p + 1] < pair_iv_off[p]) { ctx->err = "debug select: pair interval offsets decrease"; return SK_ERR_PARAM; }
    nint[p] = (uint32_t)(pair_iv_off[p + 1] - pair_iv_off[p]);
    for (uint64_t i = pair_iv_off[p]; i < pair_iv_off[p + 1]; i++) {
      const int64_t* x = intervals + 10 * i;
      bool ok = x[0] >= 0 && x[0] < (1ll << 31) && x[1] >= 0 && x[1] <= 0xFFFFFFFFll && x[8] >= 0 && x[8] < (int64_t)pair_chunks[p] &&
                (x[9] == 0 || x[9] == 1);
      for (int f = 2; f < 8; f++) ok = ok && x[f] >= 0 && x[f] <= 0xFFFFFFFFll;
      if (!ok) { ctx->err = "debug select: interval field out of range"; return SK_ERR_PARAM; }
      if (!(x[2] < x[3] && x[4] < x[5])) { ctx->err = "debug select: an interval needs q0 < q1 and r0 < r1"; return SK_ERR_PARAM; }
      iv[i] = sk::make_interval((int32_t)x[0], (uint32_t)x[1], (uint32_t)x[2], (uint32_t)x[3], (uint32_t)x[4], (uint32_t)x[5],
                                (uint32_t)x[6], (uint32_t)x[7], (uint32_t)x[8], (uint32_t)x[9]);
    }
  }
  ibase[n_pairs] = TI;
  std::vector<uint64_t> first(cbase[n_pairs] + 1, 0);
  const int rc = sk::debug_dp_select(ctx, c, k, switched, cbase, abase, ibase, {}, first, std::vector<uint32_t>(cbase[n_pairs], 0),
                                     iv, nint, false, out, pair_sums);
  if (rc != SK_OK) for (uint64_t i = 0; i < n_pairs; i++) sk_chain_debug_free(out + i);
  return rc;
}

int sk_chain_pairs_debug(sk_ctx* ctx, const sk_sketch_set* refs, const sk_sketch_set* queries, const uint64_t* pairs, uint64_t n_pairs,
                         const sk_map_params* mp, sk_chain_debug* out) {
  if (!ctx || !refs || !queries || !mp || (n_pairs && (!pairs || !out))) return SK_ERR_PARAM;
  if (n_pairs == 0) return SK_OK;
  memset(out, 0, n_pairs * sizeof(*out));
  std::vector<sk_ani_result> res(n_pairs);
  const int rc = sk::chain_impl(ctx, refs, queries, pairs, n_pairs, mp, res.data(), out, nullptr);
  if (rc != SK_OK)
    for (uint64_t i = 0; i < n_pairs; i++) sk_chain_debug_free(out + i);
  return rc;
}

int sk_chain_pair_debug(sk_ctx* ctx, const sk_sketch_set* refs, const sk_sketch_set* queries, uint64_t pair, const sk_map_params* mp,
                        sk_chain_debug* out) {
  if (!out) return SK_ERR_PARAM;
  return sk_chain_pairs_debug(ctx, refs, queries, &pair, 1, mp, out);
}

}  // extern "C"
