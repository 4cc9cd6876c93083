/* ============================================================================================
 * skani_b200.h -- C ABI of libskani_b200.so: the Hopper (H100, sm_90a) implementation of skani's
 * ANI hot path (FracMinHash seeding -> marker screen -> seed intersection / chaining / ANI+AF /
 * learned-ANI regression).
 *
 * The reference (bluenote-1577/skani v0.3.0, Rust) has no FFI layer: the boundary this header
 * replaces is the crate's public Rust API, the one tests/tests.rs:52-56 drives.  Every entry point
 * cites the reference function it stands in for (paths relative to the reference tree).  The
 * functions are batched because a GPU wants whole batches and device-resident sketches; semantics
 * per genome / per pair are exactly those of the cited functions.
 *
 * Conventions: plain pointers and sizes only; every function returns 0 on success and a negative
 * sk_status otherwise (the library never aborts the host process; the reference panics instead,
 * e.g. src/params.rs:183-185).  sk_last_error() gives a message.  A context is bound to one CUDA
 * device and is not thread-safe; use one context per host thread / per GPU.
 * There is NO CPU fallback: without a usable CUDA device sk_ctx_create fails.
 * ============================================================================================ */
#ifndef SKANI_B200_H
#define SKANI_B200_H
#include <stdint.h>
#ifdef __cplusplus
extern "C" {
#endif

typedef struct sk_ctx sk_ctx;
typedef struct sk_sketch_set sk_sketch_set; /* device-resident Vec<Sketch> (src/types.rs:253-277) */

typedef enum {
  SK_OK = 0,
  SK_ERR_CUDA = -1,    /* a CUDA runtime call failed */
  SK_ERR_PARAM = -2,   /* invalid argument (reference: panic!, src/params.rs:183-185, src/seeding.rs:239-241) */
  SK_ERR_NOMEM = -3,
  SK_ERR_STATE = -4
} sk_status;

/* src/params.rs:137-146 SketchParams (DNA members).  Requires c <= marker_c, k <= 16. */
typedef struct {
  uint32_t c;        /* FracMinHash compression, default 125 (src/params.rs:15) */
  uint32_t k;        /* seed k-mer length, default 15 (src/params.rs:17) */
  uint32_t marker_c; /* marker compression, default 1000 (src/params.rs:33) */
} sk_sketch_params;

/* The members of CommandParams (src/params.rs:96-123) that reach screen.rs / chain.rs. */
typedef struct {
  double screen_val;            /* -s as a fraction; 0 => 0.80 (src/triangle.rs:34-42) */
  double min_aligned_frac;      /* --min-af / 100; < 0 => 0.15 (src/chain.rs:101-107) */
  double both_min_aligned_frac; /* --both-min-af / 100; <= 0 disables (src/chain.rs:500-505) */
  int32_t robust;               /* --robust (src/chain.rs:428-437) */
  int32_t median;               /* --median */
  int32_t learned_ani;          /* regression on/off (src/regression.rs:8-28) */
  int32_t rescue_small;         /* !--faster-small (src/parse.rs:798) */
} sk_map_params;

/* src/types.rs:559-582 AniEstResult minus the strings (the caller owns the names).
 * Sentinels preserved: ani = NaN (no anchors / no chains, src/chain.rs:416-419), ani = -1 (AF cutoff, :500-517). */
typedef struct {
  float ani, af_query, af_ref, ci_lower, ci_upper, std;
  float q90_q, q90_r, q50_q, q50_r, q10_q, q10_r;
  uint32_t num_contigs_q, num_contigs_r, avg_chain_int_len, total_bases_covered;
  uint32_t ref_id, query_id; /* indices into the ref / query sketch sets */
} sk_ani_result;

/* ---- context ------------------------------------------------------------------------------- */
int sk_device_count(void);   /* usable CUDA devices (0 = none: nothing in this library can run) */
/* free and total memory of a device in bytes (cudaMemGetInfo), e.g. to decide whether a triangle's sketches fit it */
int sk_device_memory(int device, uint64_t* free_bytes, uint64_t* total_bytes);
int sk_ctx_create(int device, sk_ctx** out);
int sk_ctx_destroy(sk_ctx* ctx);
const char* sk_last_error(const sk_ctx* ctx);
/* number of this library's kernel launches since the context was created (for bench.py's gpu_launches) */
uint64_t sk_ctx_launch_count(const sk_ctx* ctx);
/* CUDA stream the context launches on (cudaStream_t), so callers can bracket it with events */
void* sk_ctx_stream(const sk_ctx* ctx);
/* per-kernel device timing for measurement runs: when on, every major kernel launch is bracketed with CUDA events on
 * the launch stream.  sk_ctx_get_timing writes "kernel_name total_ms launches\n" lines into buf (NUL-terminated). */
int sk_ctx_set_timing(sk_ctx* ctx, int on);
int sk_ctx_get_timing(sk_ctx* ctx, char* buf, uint64_t cap, int reset);

/* Which of the reference's two seeders the context reproduces.  SK_SEED_AVX2 (default) = avx2_seeding::avx2_fmh_seeds
 * (src/avx2_seeding.rs:33), what every x86-64 host with AVX2 runs (src/file_io.rs:196-226 dispatch): 4 quarter-lanes, the
 * last (len - 20) mod 4 windows never examined, only 'N' breaks a window, for 21 bases.  SK_SEED_SCALAR = seeding::fmh_seeds
 * (src/seeding.rs:225-323), what hosts WITHOUT AVX2 run: one lane, every window, 'N' and 'n' break the next k windows.
 * Both are bit-exact against the oracle (tests/test_gpu_seeding.py).  With SK_SEED_SCALAR sk_sketch_batch_2bit expects the
 * caller's N mask to flag 'n' as well. */
#define SK_SEED_AVX2 0
#define SK_SEED_SCALAR 1
int sk_ctx_set_seeding_semantics(sk_ctx* ctx, int semantics);

/* ---- seeding: replaces avx2_seeding::avx2_fmh_seeds (src/avx2_seeding.rs:33, the path x86-64 hosts run;
 *      bit-exact incl. its 4-lane split, dropped tail windows and 'N' rule) and the Sketch assembly of
 *      file_io::fastx_to_sketches / fastx_to_multiple_sketch_rewrite (src/file_io.rs:141-362) ------------
 * bases_ascii : the kept records' sequence bytes (ASCII, newlines already removed), concatenated
 * contig_off  : n_contigs+1 byte offsets into bases_ascii
 * genome_of_contig : non-decreasing genome index per contig, 0..n_genomes-1 (file mode: all contigs of a file
 *               share one genome; -i / --qi / --ri mode: one genome per contig).  Contig index inside a
 *               genome = rank among that genome's contigs, as src/file_io.rs:167,188,230.
 *               The >= 500 bp record filter (src/file_io.rs:176) is applied by the caller.
 * Input buffers are HOST memory (pinned or not); the call stages them to the device itself in sub-batches, converting
 * a share of every sub-batch to 2-bit on the host while the previous one is uploaded and seeded.                */
int sk_sketch_batch(sk_ctx* ctx, const uint8_t* bases_ascii, const uint64_t* contig_off, uint32_t n_contigs,
                    const uint32_t* genome_of_contig, uint32_t n_genomes, const sk_sketch_params* params,
                    sk_sketch_set** out);
/* Packed input (SURVEY.md section 8b `bases_ascii_or_2bit`): the caller already holds the sequences as 2-bit codes, the
 * reference's own in-register encoding (src/types.rs:40-49 BYTE_TO_SEQ; A 0, C 1, G 2, T/U 3, anything else 0).
 * units : contig i owns the u64 words [U_i, U_i + ceil(len_i / 32)), U_i = sum_{j<i} ceil(len_j / 32); base b of a word sits in
 *         bits 2b..2b+1 (bases past the contig end must be 0)
 * nmask : same indexing with u32 words, bit b = base b is the byte 'N' (the only byte the AVX2 seeder treats as a
 *         break, src/avx2_seeding.rs:115-126); NULL = no 'N' anywhere
 * HOST memory (pinned or not); 0.25 B/base cross PCIe instead of 1 (+ the mask words of contigs that contain 'N').
 * sk_pack_contig converts one contig's ASCII to this layout on the host (AVX-512 / AVX2 / scalar). */
int sk_pack_contig(const uint8_t* ascii, uint64_t n_bases, uint64_t* units, uint32_t* nmask);
/* name of the packing implementation this machine runs ("avx512vbmi", "avx512bw", "avx2", "scalar"); static string */
const char* sk_pack_impl(void);
int sk_sketch_batch_2bit(sk_ctx* ctx, const uint64_t* units, const uint32_t* nmask, const uint32_t* contig_len, uint32_t n_contigs,
                         const uint32_t* genome_of_contig, uint32_t n_genomes, const sk_sketch_params* params, sk_sketch_set** out);
/* share of the bases that the last sk_sketch_batch / sk_triangle on this context converted to 2-bit on the host before the
 * upload (the call adapts it to the measured packing and PCIe rates; the rest is converted by a kernel) */
double sk_ctx_last_pack_share(const sk_ctx* ctx);
/* Same, with bases_ascii already resident in DEVICE memory (bench "value" leg). contig_off / genome_of_contig stay host. */
int sk_sketch_batch_dev(sk_ctx* ctx, const uint8_t* d_bases_ascii, const uint64_t* contig_off, uint32_t n_contigs,
                        const uint32_t* genome_of_contig, uint32_t n_genomes, const sk_sketch_params* params,
                        sk_sketch_set** out);
int sk_sketch_set_free(sk_sketch_set* set);
/* append `src` to `dst` (genome ids of src shift by dst's genome count); src stays valid. Same params required. */
int sk_sketch_set_append(sk_sketch_set* dst, const sk_sketch_set* src);

uint32_t sk_sketch_set_n_genomes(const sk_sketch_set* set);
/* per-genome sizes: seed records (Sum of position-list lengths of Sketch.kmer_seeds_k), distinct seed k-mers,
 * markers (|Sketch.marker_seeds|), contigs, total_sequence_length */
int sk_sketch_set_genome_info(const sk_sketch_set* set, uint32_t genome, uint64_t* n_records, uint64_t* n_kmers,
                              uint64_t* n_markers, uint64_t* n_contigs, uint64_t* total_len);
/* Copy one genome's sketch to caller-allocated host arrays: seed records sorted by (kmer, contig, pos)
 * [kmer = SeedBits key of kmer_seeds_k, pos = SeedPosition.pos, contig_canon = SeedPosition.contig_index_canonical,
 * src/types.rs:125-138], markers ascending, contig lengths in contig order.  Any pointer may be NULL. */
int sk_sketch_set_export(const sk_sketch_set* set, uint32_t genome, uint32_t* kmer, uint32_t* pos,
                         uint32_t* contig_canon, uint64_t* markers, uint32_t* contig_lengths);
/* Build a one-genome sketch set from such arrays (e.g. decoded from a skani .sketch / sketches.db entry,
 * file_io::sketches_from_sketch src/file_io.rs:680).  Records may be in any order; markers must be distinct. */
int sk_sketch_set_import(sk_ctx* ctx, const sk_sketch_params* params, const uint32_t* kmer, const uint32_t* pos,
                         const uint32_t* contig_canon, uint64_t n_records, const uint64_t* markers, uint64_t n_markers,
                         const uint32_t* contig_lengths, uint32_t n_contigs, sk_sketch_set** out);
/* Batched form (e.g. every entry of a skani database decoded on the host: src/sketch_db.rs:104-121 get_sketch,
 * src/file_io.rs:719 marker_sketches_from_marker_file): genome g owns records [rec_off[g], rec_off[g+1]), markers
 * [mk_off[g], mk_off[g+1]) and contigs [ctg_off[g], ctg_off[g+1]) of the concatenated arrays (offset arrays have
 * n_genomes + 1 entries, n_genomes >= 1).  total_len: Sketch.total_sequence_length per genome, or NULL = sum of the
 * genome's contig lengths (marker-only sketches carry no contig lengths).  A batch is limited to < 2^31 records and
 * markers; larger databases are imported in several batches joined with sk_sketch_set_append.  Markers must be < 2^42
 * and seed k-mers < 4^k (a k-mer hash of a DNA sketch always is); SK_ERR_PARAM otherwise. */
int sk_sketch_set_import_batch(sk_ctx* ctx, const sk_sketch_params* params, uint32_t n_genomes, const uint64_t* rec_off,
                               const uint32_t* kmer, const uint32_t* pos, const uint32_t* contig_canon,
                               const uint64_t* mk_off, const uint64_t* markers, const uint64_t* ctg_off,
                               const uint32_t* contig_lengths, const uint64_t* total_len, sk_sketch_set** out);
/* Build a set of n_blobs genomes, in the order given, from skani v0.3 sketch blobs exactly as stored: a .sketch file's
 * bytes or an index.db slice of sketches.db (blob g = bytes[blob_off[g], blob_off[g] + blob_len[g]), SketchParams
 * included).  `bytes` is HOST memory (pinned or not).  The host walks each blob's framing; the k-mer map is expanded on
 * the device, records in the same order as the host decoder's, so the set equals the one sk_sketch_set_import_batch builds
 * from the decoded records (genome g: the blob's contig lengths and total_sequence_length).  Every blob's (c, k,
 * marker_c) must equal *params; amino-acid blobs are refused.  On SK_ERR_PARAM, *bad_blob (may be NULL) names the blob
 * that does not decode: the first one whose framing or parameters are refused, else the first one with a multi-position
 * index past its lists; UINT32_MAX when the error is not a blob's.  Same limits as sk_sketch_set_import_batch
 * (< 2^31 records, keys, markers and contigs per call). */
int sk_sketch_set_import_blobs(sk_ctx* ctx, const sk_sketch_params* params, const uint8_t* bytes, const uint64_t* blob_off,
                               const uint64_t* blob_len, uint32_t n_blobs, sk_sketch_set** out, uint32_t* bad_blob);

/* Genomes [g0, g0 + n) of a set encoded on the device as skani v0.3 entries, byte for byte what the host writer
 * (skani_b200/cli/sketch_db.hpp: put_params + put_sketch) writes for the same sketch:
 *   SK_ENTRY_FULL     (SketchParams, Sketch): one sketches.db entry, or a whole .sketch file
 *   SK_ENTRY_MARKERS  Sketch::get_markers_only, without params: one element of markers.bin's Vec<Sketch>
 * k-mers ascend, each with its records in (contig, pos) order.  The set gives c, k, marker_c (SketchParams; the Sketch's
 * marker_c field holds c, src/types.rs:347), total_sequence_length, contig lengths, records and markers;
 * repetitive_kmers is 0 and both flags false.  The caller gives what the set does not hold, in sk_entry_meta (entry i is
 * genome g0 + i):
 *   file_name        names[name_off[i], name_off[i + 1])
 *   contigs          contig names j in [contig_first[i], contig_first[i + 1]), name j = contig_names[contig_name_off[j],
 *                    contig_name_off[j + 1]) (written as given, independently of the set's contig lengths)
 *   contig_order     contig_order[i]
 * sk_sketch_set_encode_sizes: entry_len[i] = the length of entry i (one count pass on the device for the full form).
 * sk_sketch_set_encode: the entries back to back from out[0] (host memory, pinned or not; entry_len may be NULL).
 * g0 + n past the set, an unknown form, missing or decreasing metadata, or out_cap below the entries' total give
 * SK_ERR_PARAM.  n = 0 writes nothing.  At most 2^31 - 2 k-mers per call. */
typedef enum { SK_ENTRY_FULL = 0, SK_ENTRY_MARKERS = 1 } sk_entry_form;
typedef struct {
  const char* names;
  const uint64_t* name_off;          /* [n + 1] */
  const char* contig_names;
  const uint64_t* contig_name_off;   /* [contig_first[n] + 1] */
  const uint64_t* contig_first;      /* [n + 1] */
  const uint64_t* contig_order;      /* [n] */
} sk_entry_meta;
int sk_sketch_set_encode_sizes(const sk_sketch_set* set, uint32_t g0, uint32_t n, int form, const sk_entry_meta* meta, uint64_t* entry_len);
int sk_sketch_set_encode(const sk_sketch_set* set, uint32_t g0, uint32_t n, int form, const sk_entry_meta* meta, uint8_t* out,
                         uint64_t out_cap, uint64_t* entry_len);

/* ---- multi-GPU plumbing (the reference is single-process; SURVEY.md section 8e): a sketch set is flattened into ONE
 *      device buffer + a small host metadata vector so that ranks can exchange sketches with a single NCCL all-gather
 *      over NVLink, then rebuilt (rank-major genome order) on every GPU.
 * sk_sketch_set_blob_size: bytes of the device blob and number of u64 metadata words.
 * sk_sketch_set_pack     : d_blob (device, >= bytes) and host_meta (host, >= words) are caller-allocated.
 * sk_sketch_set_unpack   : builds ONE set from n_parts blobs (device pointers) + their metadata, concatenated in order. */
int sk_sketch_set_blob_size(const sk_sketch_set* set, uint64_t* device_bytes, uint64_t* host_meta_words);
int sk_sketch_set_pack(const sk_sketch_set* set, void* d_blob, uint64_t* host_meta);
int sk_sketch_set_unpack(sk_ctx* ctx, uint32_t n_parts, const void* const* d_blobs, const uint64_t* const* host_metas,
                         sk_sketch_set** out);
/* Subset variants for exchanges that move only what a rank needs (skani_b200/multi_gpu.py: markers of every genome are
 * all-gathered for the screen, then each rank fetches the full sketches of just the genomes its pairs touch):
 * genomes[0..n) index `set` (NULL = all genomes, in order); the blob holds them in that order.  With
 * SK_PACK_MARKERS_ONLY the blob carries the marker arrays only (enough for sk_screen_*; such a set chains to
 * "no anchors", ani = NaN).  Same blob / metadata format as sk_sketch_set_pack, so sk_sketch_set_unpack reads both. */
#define SK_PACK_MARKERS_ONLY 1
#define SK_PACK_TABLES 2   /* also carry the per-genome k-mer hash tables, so sk_sketch_set_unpack does not rebuild them */
int sk_sketch_set_subset_blob_size(const sk_sketch_set* set, const uint32_t* genomes, uint32_t n, int flags,
                                   uint64_t* device_bytes, uint64_t* host_meta_words);
int sk_sketch_set_pack_subset(const sk_sketch_set* set, const uint32_t* genomes, uint32_t n, int flags, void* d_blob,
                              uint64_t* host_meta);

/* ---- marker screen: replaces screen::kmer_to_sketch_from_refs + screen_refs / screen_refs_indices /
 *      check_markers_quickly (src/screen.rs:190, 148, 39, 84) -----------------------------------------------
 * Output pair lists are malloc'd by the library (free with sk_free), sorted ascending, each pair = (a << 32) | b. */
/* triangle: pairs (i, j), i < j, such that j is in screen_refs(i) (src/triangle.rs:71-90; asymmetric rule) */
int sk_screen_triangle(sk_ctx* ctx, const sk_sketch_set* set, const sk_map_params* mp, uint64_t** pairs_ij,
                       uint64_t* n_pairs);
/* same, restricted to rows i with i % row_mod == row_rem: the partition of the pair set over ranks (no communication) */
int sk_screen_triangle_rows(sk_ctx* ctx, const sk_sketch_set* set, const sk_map_params* mp, uint32_t row_mod, uint32_t row_rem,
                            uint64_t** pairs_ij, uint64_t* n_pairs);
/* one BLOCK of a sharded triangle screen: the pairs (i, j), i < j, g_begin <= j < g_end of sk_screen_triangle(set), computed from
 * the markers of the genomes [0, g_end) only.  The union over a partition of [0, n) into blocks is sk_screen_triangle's list
 * (multi-GPU: every GPU screens the rows of its own genome block against everything before them, src/triangle.rs:71-90). */
int sk_screen_triangle_block(sk_ctx* ctx, const sk_sketch_set* set, uint32_t g_begin, uint32_t g_end, const sk_map_params* mp,
                             uint64_t** pairs_ij, uint64_t* n_pairs);
/* dist / search: pairs (ref, query).  mode 0 = check_markers_quickly with rescue_small from mp (dist without index,
 * src/dist.rs:104), mode 1 = check_markers_quickly with rescue_small = false (search, src/search.rs:127),
 * mode 2 = screen_refs via the inverted index (dist with index, src/dist.rs:122), mode 3 = screen_refs_indices
 * (search with index, src/search.rs:134). */
int sk_screen_query_ref(sk_ctx* ctx, const sk_sketch_set* refs, const sk_sketch_set* queries, const sk_map_params* mp,
                        int mode, uint64_t** pairs_rq, uint64_t* n_pairs);
void sk_free(void* p);

/* ---- persistent reference marker index (search over query groups): the references' markers sorted once, then any
 *      number of query sets screened against them without re-sorting the references.
 * sk_ref_index_screen(ctx, idx, queries, mp, mode) returns exactly sk_screen_query_ref(ctx, refs, queries, mp, mode): the
 * same sorted (ref << 32 | query) list for modes 0-3, query ids local to `queries`.  The index lives on the context that
 * created it (the CLI's ctxs[0]); the queries must be on that context too, and refs may be freed once it is created.
 * Device memory: 12 bytes per reference marker (the sorted marker and its reference), 8 bytes per reference and 256 KiB
 * of prefix buckets per part; creating a part also takes about 16 bytes per marker of the part in temporaries.  The
 * references are cut into contiguous parts of < 2^31 markers (SK_REF_INDEX_PART_MARKERS, read at creation, lowers the
 * bound); a query set is screened against each part in turn, so databases of 2^31 markers and more are screened too.
 * A screen takes 8 bytes per query marker (the lookup slices) besides its pair buffer. */
typedef struct sk_ref_index sk_ref_index;
int sk_ref_index_create(sk_ctx* ctx, const sk_sketch_set* refs, sk_ref_index** idx);
int sk_ref_index_screen(sk_ctx* ctx, const sk_ref_index* idx, const sk_sketch_set* queries, const sk_map_params* mp, int mode,
                        uint64_t** pairs_rq, uint64_t* n_pairs);
/* references indexed, parts, device bytes held (any pointer may be NULL) */
int sk_ref_index_info(const sk_ref_index* idx, uint32_t* n_refs, uint32_t* n_parts, uint64_t* device_bytes);
int sk_ref_index_free(sk_ref_index* idx);

/* ---- chaining: replaces chain::map_params_from_sketch + chain::chain_seeds (src/chain.rs:88, 144) and
 *      regression::get_model / predict_from_ani_res (src/regression.rs:12, 30) for every listed pair ---------
 * pairs[i] = (ref_index << 32) | query_index; out[i] is the AniEstResult of chain_seeds(refs[ref], queries[query]).
 * file-name tie-break of switch_qr (src/chain.rs:19-21): name(x) > name(y) iff its `name_rank` is larger, equal ranks =
 * equal file names.  Default rank = index in the set (one file per sketch, sets built in sorted file order,
 * src/file_io.rs:250); callers sketching individual records (-i / --qi / --ri) MUST give the records of one file equal
 * ranks with sk_sketch_set_set_name_ranks; for two different sets the query set ranks after the ref set by default. */
int sk_chain_pairs(sk_ctx* ctx, const sk_sketch_set* refs, const sk_sketch_set* queries, const uint64_t* pairs,
                   uint64_t n_pairs, const sk_map_params* mp, sk_ani_result* out);
int sk_sketch_set_set_name_ranks(sk_sketch_set* set, const uint64_t* ranks /* n_genomes */);

/* ---- mappings: where each pair aligns.  One record per chain interval that the non-overlap selection kept
 *      (get_nonoverlapping_chains, src/chain.rs:1008-1099), joined to the identity estimate of the chunk it was chained in. */
typedef struct {
  uint32_t query_contig, ref_contig;  /* contig indices in the pair's query / reference genome (caller's orientation) */
  uint32_t q0, q1, r0, r1;            /* first / last anchor seed position of the chain on each side, as the chain holds them */
  uint32_t num_anchors, chunk;        /* anchors in the chain; the pair-local chunk it was chained in */
  double   chunk_est;                 /* that chunk's identity estimate (raw, before the learned-ANI regression); 0 if none */
  uint32_t chunk_weight;              /* its weight; 0 if none */
  uint8_t  reverse, switched, chunk_valid, pad;  /* chunk_valid: 0 no estimate, 1 estimate, 3 estimate after the
                                                    putative-ANI filter.  switched = 1: the chunks are windows of the reference */
} sk_mapping;                         /* 48 bytes */
/* sk_chain_pairs plus the mappings of every pair.  out is byte for byte sk_chain_pairs' out for the same arguments.  Pair i
 * owns (*maps)[map_off[i] .. map_off[i + 1]) (map_off: n_pairs + 1 entries, caller-allocated; *maps malloc'd, sk_free):
 * every interval the selection kept for it, whatever its ani (NaN and -1 included), sorted by (query_contig, q0, q1,
 * ref_contig, r0, r1, reverse, chunk).  A seed position is the index of the last base of its k-mer, so a record covers bases
 * [q0 - k + 1, q1 + 1) of its query contig and [r0 - k + 1, r1 + 1) of its reference contig. */
int sk_chain_pairs_mappings(sk_ctx* ctx, const sk_sketch_set* refs, const sk_sketch_set* queries, const uint64_t* pairs,
                            uint64_t n_pairs, const sk_map_params* mp, sk_ani_result* out, uint64_t* map_off,
                            sk_mapping** maps);

/* parity taps (test use), per pair: all outputs are malloc'd (sk_chain_debug_free). anchors: 5 x u32 per anchor
 * (query_contig, query_pos, ref_contig, ref_pos, reverse) in sorted order (src/chain.rs:721); chunk_first: n_chunks+1;
 * score/pointer per anchor (chunk-local pointer, src/chain.rs:881-882); intervals: 11 x i64 per interval in the
 * descending order of src/chain.rs:1012: score,num_anchors,q0,q1,r0,r1,ref_contig,query_contig,chunk,reverse,kept;
 * ests: sorted (est, weight) of src/chain.rs:414; chunk_stats: 9 x u32 per chunk (src/chain.rs:204-394): total_anchors, rq0,
 * rq1 (min q0 / max q1 of the kept intervals; 0xFFFFFFFF / 0 without one), tbcq (total_bases_contained_query, wrapping),
 * n_int (kept intervals), n_seeds, num_in (seeds inside the intervals padded by c), upper_lower (seeds in [rq0, rq1]),
 * filtered (1 = the putative-ANI filter replaced the weight n_seeds by upper_lower). */
typedef struct {
  sk_ani_result result;
  int32_t switched;
  uint64_t n_anchors, n_chunks, n_intervals, n_ests;
  uint32_t* anchors;
  uint32_t* chunk_first;
  uint32_t* chunk_nseeds;
  int64_t* score;
  uint32_t* pointer;
  int64_t* intervals;
  double* est;
  uint64_t* weight;
  uint32_t* chunk_stats;
} sk_chain_debug;
/* sk_chain_pairs_debug runs the batching, pair descriptors and kernel instantiations of sk_chain_pairs on the same pair list
 * (the kernels additionally store the per-anchor DP scores and pointers) and fills out[i] from pair i's slices of the batch.
 * On error every out[i] is freed.  sk_chain_pair_debug is its one-pair call. */
int sk_chain_pairs_debug(sk_ctx* ctx, const sk_sketch_set* refs, const sk_sketch_set* queries, const uint64_t* pairs,
                         uint64_t n_pairs, const sk_map_params* mp, sk_chain_debug* out /* n_pairs */);
int sk_chain_pair_debug(sk_ctx* ctx, const sk_sketch_set* refs, const sk_sketch_set* queries, uint64_t pair,
                        const sk_map_params* mp, sk_chain_debug* out);
void sk_chain_debug_free(sk_chain_debug* d);
/* (test use) the device's per-chunk identity, chunk_estimate of chunkstat_kernel, over n chunks given as 8 x u32 each:
 * total_anchors, rq0, rq1, tbcq, n_int, n_seeds, num_in, upper_lower (host arrays).  Per chunk: est, weight, and valid =
 * 0 (no estimate), 1 (estimate) or 3 (estimate, the putative-ANI filter applied). */
int sk_debug_chunk_estimate(sk_ctx* ctx, uint64_t n, const uint32_t* inputs, uint32_t c, uint32_t k, double* est,
                            uint32_t* weight, uint32_t* valid);
/* (test use) the chain back end's DP and interval selection on given anchors (host arrays).  Pair p owns the chunks
 * pair_chunk_off[p] .. pair_chunk_off[p + 1], chunk i the anchors chunk_anchor_off[i] .. chunk_anchor_off[i + 1] (both offset
 * arrays start at 0), 5 x u32 per anchor as in sk_chain_debug.  A chunk holds at least one anchor, all of one query contig,
 * sorted by (query_pos, ref_contig, ref_pos, reverse) as the chunking kernel emits them; ref contigs are < 2^30 and positions
 * < 2^32 - 65536; anything else is refused (SK_ERR_PARAM with a message).  The workspace is filled as sk_chain_pairs' chunking
 * leaves it (interval capacity floor(anchors / 3) per pair), and the DP instantiation sk_chain_pairs chooses for c (with the
 * same SK_DP_* environment hooks) and the interval selection run on it.  out[p] receives anchors, chunk_first, score,
 * pointer, the sorted intervals with kept flags and chunk_stats, whose first five fields are the selection's per-chunk sums
 * (the seed counts are 0, result and ests are empty); pair_sums[2p] / [2p + 1] = the kept intervals' summed
 * (q1 - q0) + 2c + k (wrapping) and their number.  switched[p] != 0: tbcq sums ref spans.  At most 65535 pairs. */
int sk_debug_chain_anchors(sk_ctx* ctx, uint32_t c, uint32_t k, uint64_t n_pairs, const uint64_t* pair_chunk_off,
                           const uint64_t* chunk_anchor_off, const uint32_t* anchors, const uint32_t* switched,
                           sk_chain_debug* out /* n_pairs */, uint32_t* pair_sums /* 2 x n_pairs */);
/* (test use) the interval selection alone on given intervals: pair p owns intervals pair_iv_off[p] .. pair_iv_off[p + 1]
 * (10 x i64: score, num_anchors, q0, q1, r0, r1, ref_contig, query_contig, chunk, reverse; any order; q0 < q1, r0 < r1,
 * chunk < pair_chunks[p], 0 <= score < 2^31, other fields u32) and pair_chunks[p] chunks; the interval capacity is the list's
 * length.  Outputs as sk_debug_chain_anchors, without anchors. */
int sk_debug_select_intervals(sk_ctx* ctx, uint32_t c, uint32_t k, uint64_t n_pairs, const uint64_t* pair_iv_off,
                              const int64_t* intervals, const uint32_t* pair_chunks, const uint32_t* switched,
                              sk_chain_debug* out /* n_pairs */, uint32_t* pair_sums /* 2 x n_pairs */);
/* (test use) sk_dereplicate's marker index and row screen on given genome lists.  Slot s of the index holds genome
 * slot_genome[s] of set (markers only are read); the slots join it in n_batches index additions of batch_sizes[b] genomes
 * each (summing to n_slots), as the waves add representatives, merging each batch into the keys built so far.  Then rows
 * (genome ids) are screened against the index: upper = 0 screens every slot, which gives the triangle's screen pairs with one
 * genome in rows and the other in slot_genome when the two lists share no genome; upper != 0 screens row k against the slots
 * above k, which requires rows == slot_genome and gives the triangle's pairs inside the list.  *pairs (malloc'd, sk_free;
 * never NULL) receives the *n_pairs passing pairs as min << 32 | max, sorted.  keys / n_keys (may both be NULL): the index's
 * keys, marker << 22 | slot, ascending (malloc'd, sk_free).  bucket (may be NULL): its 2^16 + 1 prefix buckets.  Refusals
 * (SK_ERR_PARAM with a message): NULL arguments, a genome id >= the set's genomes, batch sizes not summing to n_slots,
 * upper with rows other than slot_genome, and sk_dereplicate's index limits (more than 2^22 - 1 slots, 2^31 or more keys). */
int sk_debug_derep_screen(sk_ctx* ctx, const sk_sketch_set* set, const sk_map_params* mp, const uint32_t* slot_genome,
                          uint32_t n_slots, const uint32_t* batch_sizes, uint32_t n_batches, const uint32_t* rows, uint32_t n_rows,
                          int upper, uint64_t** pairs, uint64_t* n_pairs, uint64_t** keys /* may be NULL */,
                          uint64_t* n_keys /* may be NULL */, uint32_t* bucket /* 2^16 + 1, may be NULL */);

/* ---- whole triangle (src/triangle.rs:13-105: sketch -> screen -> chain -> keep ani > 0.1) from HOST sequence
 *      buffers; results malloc'd (sk_free).  Timing breakdown (seconds, device events) optional. -------------- */
typedef struct {
  double t_sketch, t_screen, t_chain, t_total;
  uint64_t n_pairs_screened, n_pairs_kept;
} sk_triangle_stats;
int sk_triangle(sk_ctx* ctx, const uint8_t* bases_ascii, const uint64_t* contig_off, uint32_t n_contigs,
                const uint32_t* genome_of_contig, uint32_t n_genomes, const sk_sketch_params* sp,
                const sk_map_params* mp, sk_ani_result** out, uint64_t* n_out, sk_triangle_stats* stats);

/* (sk_triangle and sk_triangle_local also accept a DEVICE pointer for bases_ascii: genomes already resident in HBM go through the
 * same seed || screen || chain pipeline without the pack / upload stages.) */
/* Same, and additionally hands back the device-resident sketch set of all n_genomes genomes (with their k-mer tables), e.g.
 * to chain further pairs against it (the cross-block pairs of a multi-GPU run).  name_ranks: optional file-name order per
 * genome for the switch_qr tie-break (see sk_sketch_set_set_name_ranks), NULL = index order.  Free with sk_sketch_set_free. */
int sk_triangle_local(sk_ctx* ctx, const uint8_t* bases_ascii, const uint64_t* contig_off, uint32_t n_contigs,
                      const uint32_t* genome_of_contig, uint32_t n_genomes, const sk_sketch_params* sp,
                      const sk_map_params* mp, const uint64_t* name_ranks, sk_ani_result** out, uint64_t* n_out,
                      sk_triangle_stats* stats, sk_sketch_set** set_out);

/* sk_triangle_local for callers whose genomes are already 2-bit packed on the host (sk_sketch_batch_2bit's layout: units of 32
 * bases, optional 'N' mask, contig lengths): 0.25 B/base leave host memory instead of 1 -- with several GPUs per host the ASCII
 * form is bounded by the host's memory bandwidth (DESIGN.md section 4).  set_out may be NULL. */
int sk_triangle_2bit(sk_ctx* ctx, const uint64_t* units, const uint32_t* nmask, const uint32_t* contig_len, uint32_t n_contigs,
                     const uint32_t* genome_of_contig, uint32_t n_genomes, const sk_sketch_params* sp, const sk_map_params* mp,
                     const uint64_t* name_ranks, sk_ani_result** out, uint64_t* n_out, sk_triangle_stats* stats,
                     sk_sketch_set** set_out);

/* ---- multi-GPU triangle from ONE host process (SURVEY.md section 8e; north_star: host -> C-ABI shim -> one exchange of the
 *      per-GPU sketch blocks over NVLink).  ctxs[0..n_ctx): one context per GPU (created with sk_ctx_create(device)); a
 *      device may appear more than once (the exchange then stays on that device: how a 1-GPU box tests this path).
 *      Genomes are split into contiguous blocks balanced by bases; every GPU runs the pipelined triangle on its block,
 *      the MARKERS of all blocks are exchanged GPU-to-GPU and screened everywhere, and the cross-block pairs are cut into
 *      equal slices whose sketches (with k-mer tables) are fetched from the owning GPUs.  Same result SET as sk_triangle
 *      (row order differs; the reference's own sparse output order is arbitrary).  results: malloc'd (sk_free). */
int sk_triangle_multi(sk_ctx* const* ctxs, uint32_t n_ctx, const uint8_t* bases_ascii, const uint64_t* contig_off, uint32_t n_contigs,
                      const uint32_t* genome_of_contig, uint32_t n_genomes, const sk_sketch_params* sp,
                      const sk_map_params* mp, const uint64_t* name_ranks, sk_ani_result** out, uint64_t* n_out,
                      sk_triangle_stats* stats);

/* ---- dist / search over several GPUs from ONE host process (src/dist.rs:98-144 screen + chain of every (ref, query) pair;
 *      src/search.rs:119-247 the same against a sketched database).  The references are split into contiguous blocks, one
 *      per context; the query set is copied to every context.  A pair's screen decision (its own marker counts,
 *      src/screen.rs:84-189) and its chain result depend on that pair alone, so the results are byte-identical to the
 *      single-context calls.  ctxs[d] may share a device.  If any context fails the call fails and sk_last_error(ctxs[0])
 *      carries that context's message. */
/* Copy a set (records, views, markers, contig tables, k-mer hash tables, name ranks) to another context, which may be on
 * another device or the same one: a packed blob with the tables (no table rebuild, except the bucket index of genomes too
 * large for a table), a peer or device copy, then an unpack.  The copy chains and screens exactly like the source. */
int sk_sketch_set_copy(sk_ctx* dst, const sk_sketch_set* src, sk_sketch_set** out);
/* References split into contiguous blocks: refs[d] lives on ctxs[d] and holds global refs [ref_first[d], ref_first[d] + G_d).
 * ref_first must be ascending and the blocks disjoint.  refs[d] may be NULL or hold 0 genomes.
 * queries[d] lives on ctxs[d] and is the same query set on every context (made with sk_sketch_set_copy).
 * Arguments that break these rules, and sets whose sketch parameters differ, give SK_ERR_PARAM.
 *   = sk_screen_query_ref on one set holding all refs: same modes 0-3, sorted, global ref ids. */
int sk_screen_query_ref_multi(sk_ctx* const* ctxs, uint32_t n_ctx, const sk_sketch_set* const* refs, const uint32_t* ref_first,
                              const sk_sketch_set* const* queries, const sk_map_params* mp, int mode,
                              uint64_t** pairs_rq, uint64_t* n_pairs);
/* pairs are global (ref << 32 | query), in any order; a pair whose ref lies in no block or whose query is out of range gives
 * SK_ERR_PARAM.  out[i] = sk_chain_pairs(one context holding all refs, pairs[i]), with ref_id global.  Default name ranks
 * (sk_sketch_set_set_name_ranks never called) are those of that one set: global ref ids, queries after all
 * ref_first[n_ctx-1] + G_{n_ctx-1} refs. */
int sk_chain_pairs_multi(sk_ctx* const* ctxs, uint32_t n_ctx, const sk_sketch_set* const* refs, const uint32_t* ref_first,
                         const sk_sketch_set* const* queries, const uint64_t* pairs, uint64_t n_pairs,
                         const sk_map_params* mp, sk_ani_result* out);
/* sk_chain_pairs_multi plus mappings as sk_chain_pairs_mappings: each context's records are merged back into pair order. */
int sk_chain_pairs_multi_mappings(sk_ctx* const* ctxs, uint32_t n_ctx, const sk_sketch_set* const* refs, const uint32_t* ref_first,
                                  const sk_sketch_set* const* queries, const uint64_t* pairs, uint64_t n_pairs,
                                  const sk_map_params* mp, sk_ani_result* out, uint64_t* map_off, sk_mapping** maps);

/* ---- triangle beyond one GPU's memory: sketches live in pinned HOST memory and come back to the device in working sets --
 * A store holds sketches with their k-mer tables, genome-indexed, in fixed-size pinned, device-mapped host slabs.
 * sk_sketch_store_add     : appends set's genomes (ids continue after the store's; name ranks continue after its largest
 *                           rank, as sk_sketch_set_append does).  Different sketch parameters give SK_ERR_PARAM.  The caller
 *                           may free the set afterwards: device memory then holds one batch of sketches at a time.
 * sk_sketch_store_genome_bytes : device bytes genome g takes in a working set (records, k-mer groups, markers, contig
 *                           tables and its k-mer hash table).
 * sk_sketch_store_set_name_ranks : file-name order of every genome (switch_qr tie-break, see sk_sketch_set_set_name_ranks).
 * sk_sketch_store_gather  : a device set on ctx holding genomes[0..n) in list order (ascending, no duplicates, < n_genomes;
 *                           anything else gives SK_ERR_PARAM), with the store's name ranks.  One batched copy pulls the
 *                           genomes' slices from the mapped host slabs over PCIe; the k-mer tables come along (genomes of
 *                           2^20 or more records carry none and get the bucket index rebuilt, as sk_sketch_set_unpack does).
 *                           flags = SK_PACK_MARKERS_ONLY gathers the markers only (enough for sk_screen_*).  A gathered set
 *                           chains, screens and exports exactly like the set that was added. */
typedef struct sk_sketch_store sk_sketch_store;
int sk_sketch_store_create(const sk_sketch_params* sp, sk_sketch_store** out);
int sk_sketch_store_add(sk_sketch_store* st, const sk_sketch_set* set);
uint32_t sk_sketch_store_n_genomes(const sk_sketch_store* st);
uint64_t sk_sketch_store_genome_bytes(const sk_sketch_store* st, uint32_t g);
int sk_sketch_store_set_name_ranks(sk_sketch_store* st, const uint64_t* ranks /* n_genomes */);
int sk_sketch_store_gather(sk_ctx* ctx, const sk_sketch_store* st, const uint32_t* genomes, uint32_t n, int flags,
                           sk_sketch_set** out);
int sk_sketch_store_free(sk_sketch_store* st);

/* sk_triangle_store: the triangle (src/triangle.rs:71-105) of every genome of a store.  The markers of all genomes are gathered
 * on ctxs[0] and screened (sk_screen_triangle); the pairs are planned into working sets whose genomes fit device_budget bytes
 * (per context; 0 = derived from the free device memory) -- components of the pair graph packed first-fit decreasing, a
 * component over budget cut into chunks of budget / 2 and chained chunk pair by chunk pair -- and the contexts take the
 * working sets in plan order: gather, sk_chain_pairs, keep ani > 0.1.  Two contexts on one device overlap one's gather with
 * the other's chaining.  Results (malloc'd, sk_free) are sorted by (ref_id, query_id) and equal sk_triangle's on the same
 * genomes and name ranks.  A genome over budget / 2 gives SK_ERR_NOMEM before any device work.  If any context fails the
 * call fails and sk_last_error(ctxs[0]) carries that context's message.  SK_TRACE=1 prints one line per working set.
 * stats (optional): t_screen = marker gather + screen; t_gather / t_chain = seconds spent gathering / chaining working sets,
 * summed over contexts; gathered_bytes = working-set bytes pulled from the store. */
typedef struct {
  uint32_t n_working_sets, n_split_components;
  uint64_t gathered_bytes, max_working_set_bytes;
  double t_screen, t_gather, t_chain;
} sk_store_stats;
int sk_triangle_store(sk_ctx* const* ctxs, uint32_t n_ctx, const sk_sketch_store* st, const sk_map_params* mp,
                      uint64_t device_budget, sk_ani_result** out, uint64_t* n_out, sk_store_stats* stats);

/* sk_query_ref_store: dist (src/dist.rs:98-144) of every (reference, query) pair of two stores.  Returns what one context
 * computes from sets R and Q holding every genome of refs and queries with the stores' name ranks:
 * sk_screen_query_ref(R, Q, mode), sk_chain_pairs(R, Q, pairs), keep ani > 0.1 (src/dist.rs:115,139).  ref_id / query_id are
 * store genome ids; results (malloc'd, sk_free) are sorted by (ref_id, query_id).  The markers of both stores are gathered on
 * ctxs[0] and screened; the pairs are planned into working sets that each hold some references and some queries within
 * device_budget bytes per context (0 = derived as in sk_triangle_store); the contexts, on one device or several, take the
 * working sets in plan order and gather each one's references from refs and queries from queries.  refs == queries (a set
 * against itself) is allowed.  A genome over budget / 2 on either side gives SK_ERR_NOMEM before any device work; stores with
 * different sketch parameters, a mode outside 0-3, NULL arguments or a context listed twice give SK_ERR_PARAM.  If any
 * context fails the call fails and sk_last_error(ctxs[0]) carries that context's message.  SK_TRACE=1 prints one line per
 * working set.  stats as in sk_triangle_store.
 * Name ranks: both stores' ranks are used exactly as stored, so the caller ranks both sides in one file-name order (set both
 * with sk_sketch_store_set_name_ranks).  Two stores left at their default ranks do NOT reproduce sk_chain_pairs' default for
 * two sets, where the queries rank after the references: both stores then rank from 0. */
int sk_query_ref_store(sk_ctx* const* ctxs, uint32_t n_ctx, const sk_sketch_store* refs, const sk_sketch_store* queries,
                       const sk_map_params* mp, int mode, uint64_t device_budget, sk_ani_result** out, uint64_t* n_out,
                       sk_store_stats* stats);

/* ---- clustering of a triangle's results (what the reference leaves to scripts/clustermap_triangle.py or a host loop over
 *      `triangle` output): genomes 0..n_genomes-1, results as sk_triangle / sk_triangle_store / sk_triangle_multi return them.
 * Edges: the rows with ani > 0.1 (the rows `triangle -E` prints) and ani >= min_ani (a float comparison: ani == min_ani is an
 * edge; NaN and -1 never are) join ref_id and query_id; the graph is undirected.  rank[g] is a permutation of 0..n-1, rank 0
 * the first choice as a representative.
 *   greedy (single_linkage = 0): genomes are visited in rank order and become representatives unless they have an edge to a
 *     representative already chosen; every other genome is assigned to its representative neighbour of highest ANI, ties to
 *     the smaller rank (that neighbour may rank after it).
 *   single linkage: clusters are the connected components; a component's representative is its member of smallest rank.
 * rep[g] = g's representative (g itself for a representative); cluster[g] = its cluster id, representatives numbered 0..C-1
 * in rank order; edge[g] = the index in results of the row joining g to rep[g], UINT64_MAX for representatives and for
 * single-linkage members not adjacent to their representative.  The outputs are a function of (edges, rank, method) alone.
 * An id >= n_genomes, a self pair, a pair listed twice among the edges, a rank that is not a permutation, a NaN min_ani or
 * NULL outputs give SK_ERR_PARAM with a message; edges that do not fit the device, or more than 2^30 - 1 of them, give
 * SK_ERR_NOMEM.  n_genomes = 0 and inputs without edges are valid.  results is HOST memory (pinned or not), uploaded in
 * chunks.
 * stats (may be NULL): edges, clusters, rounds (greedy decision rounds or single-linkage hook passes) and t_device, the
 * seconds from the first upload to the last read-back. */
typedef struct {
  float min_ani;           /* as a fraction, e.g. 0.95 */
  int32_t single_linkage;  /* 0 = greedy representatives */
} sk_cluster_params;
typedef struct {
  uint64_t n_edges;
  uint32_t n_clusters, rounds;
  double t_device;
} sk_cluster_stats;
int sk_cluster(sk_ctx* ctx, uint32_t n_genomes, const sk_ani_result* results, uint64_t n_results, const uint32_t* rank,
               const sk_cluster_params* cp, uint32_t* rep, uint32_t* cluster, uint64_t* edge, sk_cluster_stats* stats /* may be NULL */);

/* ---- average (UPGMA) and complete linkage of a triangle's results (what the reference's scripts/clustermap_triangle.py
 *      does with scipy on the dense 100 - ANI matrix), from the edge list alone.  Inputs as for sk_cluster.
 * Edges: every row with ani > 0.1 (the rows `triangle -E` prints; NaN and -1 never are); min_ani does NOT filter them, it
 * is only the cut.  A pair of genomes without an edge has similarity 0.  q = ani * 2^27 is an exact integer for every
 * float in (0.1, 2); a row with ani >= 2 (or +inf) is refused, and so is min_ani outside (0.1, 1].
 * Value of a cluster pair (A, B), P = |A| |B|: average S / (P 2^27) with S = sum of q over the edges between A and B;
 * complete min q / 2^27 when all P member pairs are edges, otherwise 0.  Values are compared exactly (128-bit
 * cross-multiplication).  A cluster's id is its smallest member rank; its best partner has the largest value, ties to the
 * smaller partner id.
 * Rounds: every active cluster finds its best partner; every pair that are each other's best partner and whose value is
 * >= q(min_ani) (in dendrogram mode: > 0) merges; clusters with no partner that could still qualify are deactivated; the
 * rounds end when none is left.  For inputs without ties the merges are those of sequential HAC (scipy's); with ties this
 * round procedure is the definition, and it is deterministic.
 * Flat clusters are the merges with value >= the cut, whatever the mode: rep[g] = the member of smallest rank, cluster[g]
 * = clusters numbered in rank order of their representatives, edge[g] = the index of the row joining g and rep[g],
 * UINT64_MAX for none.
 * Dendrogram (dendrogram != 0; merges has n_genomes - 1 rows, may be NULL otherwise): a scipy linkage matrix.  Genomes are
 * 0..n-1 in genome-index order, row j's cluster is n + j, a < b.  Rows are sorted by (value descending, round, id);
 * height = 1 - S / ldexp(P, 27) (average) or 1 - ldexp(min q, -27) (complete), rounded to nearest; the clusters left at
 * the end (no pair with value > 0 between them) are joined at height exactly 1.0 in id order, ((r0 r1) r2) ...
 * stats (may be NULL): edges, flat clusters, rounds (the rounds that merged something) and t_device.
 * Refusals as for sk_cluster, plus ani >= 2, min_ani out of range or NaN, a method other than 0 / 1 and NULL merges in
 * dendrogram mode (SK_ERR_PARAM); more than n rounds give SK_ERR_STATE. */
typedef struct {
  float min_ani;       /* the cut, as a fraction in (0.1, 1] */
  int32_t method;      /* SK_LINKAGE_AVERAGE or SK_LINKAGE_COMPLETE */
  int32_t dendrogram;  /* 1 = every merge with value > 0, written to merges */
} sk_linkage_params;
#define SK_LINKAGE_AVERAGE 0
#define SK_LINKAGE_COMPLETE 1
typedef struct {
  uint32_t a, b;   /* the joined clusters: genome index < n_genomes, or n_genomes + row */
  double height;   /* 1 - similarity */
  uint64_t size;   /* genomes in the new cluster */
} sk_merge;
int sk_cluster_linkage(sk_ctx* ctx, uint32_t n_genomes, const sk_ani_result* results, uint64_t n_results, const uint32_t* rank,
                       const sk_linkage_params* lp, uint32_t* rep, uint32_t* cluster, uint64_t* edge, sk_merge* merges,
                       sk_cluster_stats* stats /* may be NULL */);

/* ---- neighbour-joining tree of a triangle's results (what users otherwise get by printing `--full-matrix --distance` and
 *      running quicktree or rapidnj on it).  Inputs and refusals as for sk_cluster_linkage, plus: a row with ani > 1 gives
 *      SK_ERR_PARAM (its distance would be negative).  results is HOST memory.
 * Distances: d(i,j) = 1 - (double)ani for every row with ani > 0.1 (exact: such a float is a multiple of 2^-27), 1.0 for a
 * pair without one, d(i,i) = 0; R_i = sum_j d(i,j) (exact for n < 2^26).  A node's id is the smallest genome index among
 * its leaves; live nodes are ordered by id.  While m > 2 nodes are live, in float64 with every operation rounded on its own:
 *   Q = ((m-2) d_ij - R_i) - R_j over live pairs i < j; the join is the smallest Q, ties to the smallest (i, j);
 *   delta_i = 0.5 d_ij + (R_i - R_j) / (2.0 (m-2)), delta_j = d_ij - delta_i;
 *   for every other live k: d_uk = 0.5 ((d_ik + d_jk) - d_ij), R_k = ((R_k - d_ik) - d_jk) + d_uk;
 *   R_u = 0.5 ((R_i + R_j) - m d_ij); the new node u takes i's id and j leaves.
 * joins (n_genomes - 1 rows; may be NULL for n < 2): row t = (a, b, delta_i, delta_j), nodes numbered the scipy way (leaves
 * 0..n-1, row t creates n + t), a the node of smaller id.  Row n - 2 joins the last two nodes with len_a = len_b = d / 2: a
 * binary tree rooted at the midpoint of the last edge.  Branch lengths may be negative; they are returned as computed.
 * The device holds the n x n float64 matrix plus a compacted copy (at most 8 n^2 (1 + 9/16) bytes); more than fits gives
 * SK_ERR_NOMEM with the bytes needed.
 * stats (may be NULL): edges, joins written, compactions of the matrix and t_device. */
typedef struct {
  uint32_t a, b;        /* the joined nodes: genome index < n_genomes, or n_genomes + row */
  double len_a, len_b;  /* branch lengths from the new node to a and to b (distance, 1 - ANI scale) */
} sk_nj_join;
typedef struct {
  uint64_t n_edges;
  uint32_t joins, compactions;
  double t_device;
} sk_nj_stats;
int sk_neighbor_joining(sk_ctx* ctx, uint32_t n_genomes, const sk_ani_result* results, uint64_t n_results, sk_nj_join* joins,
                        sk_nj_stats* stats /* may be NULL */);
/* sk_neighbor_joining with the matrix split over n_ctx contexts (distinct devices, or several contexts on one device):
 * joins and stats (but t_device) are byte for byte sk_neighbor_joining(ctxs[0], ...)'s for any n_ctx >= 1.  Each context
 * holds full rows of a band of slots, about 8 n^2 (1 + 9/16) / n_ctx bytes; the contexts exchange the step's minima and two
 * columns (16 bytes per live node) through peer copies.  The edges are built on ctxs[0], with sk_neighbor_joining's
 * refusals and messages there.  NULL or repeated contexts give SK_ERR_PARAM, and a failure on context d is reported on
 * ctxs[0] as "context d: ...".  One host thread drives every context. */
int sk_neighbor_joining_multi(sk_ctx* const* ctxs, uint32_t n_ctx, uint32_t n_genomes, const sk_ani_result* results, uint64_t n_results,
                              sk_nj_join* joins, sk_nj_stats* stats /* may be NULL */);

/* ---- greedy dereplication of an in-memory sketch set (what galah and dRep do on top of skani): sk_cluster's greedy
 *      representatives without the triangle.  Only genome x representative pairs are screened and chained.
 * Contract: for any set (with its name ranks), mp, rank permutation and min_ani, rep[] and cluster[] equal those of
 * sk_cluster (single_linkage = 0, same min_ani and rank) run on the rows of sk_screen_triangle + sk_chain_pairs over the same
 * set, and for every member g, join[g] is byte for byte the row sk_cluster's edge[g] points to.  For a representative,
 * join[g] is all zero but ani = NaN and ref_id = query_id = g.  The result does not depend on dp->wave.
 * Exactness rests on two facts: a pair's chain result depends only on the pair, the set, its name ranks and mp; and the greedy
 * outcome depends only on the edges that touch a representative.  Every pair is screened with the triangle's rule (the
 * smaller genome index is screen_refs' query, so only its marker count can rescue the pair) and chained as (min << 32 | max).
 * Algorithm: genomes are visited in rank order in waves of dp->wave genomes (0 = the library default: 64 genomes, doubling per wave up to 4096).  A wave is
 * screened and chained against the representatives chosen so far (a wave genome with an edge to one is a member), then the
 * wave's undecided genomes against each other, decided by sk_cluster's greedy rounds; the new representatives' markers join
 * the index.  Finally every member is screened against all representatives and the pairs not chained yet are chained; each
 * member takes its representative neighbour of highest ANI, ties to the smaller rank.
 * Refusals (SK_ERR_PARAM with a message): NULL arguments, a rank that is not a permutation, a NaN min_ani, more than
 * 2^22 - 1 representatives (or undecided genomes in one wave) in an index, or 2^31 or more markers in one.  The set must be
 * one context's in-memory set; a host sketch store goes to sk_dereplicate_store.
 * stats (may be NULL): pairs that passed a screen, pairs chained, edges among the chained rows, clusters, waves, greedy rounds,
 * and the seconds spent screening, chaining, deciding (greedy rounds and assignment) and in all. */
typedef struct {
  float min_ani;   /* as a fraction, e.g. 0.95 */
  uint32_t wave;   /* genomes per wave; 0 = library default */
} sk_derep_params;
typedef struct {
  uint64_t pairs_screened, pairs_chained, n_edges;
  uint32_t n_clusters, waves, rounds;
  double t_screen, t_chain, t_decide, t_total;
} sk_derep_stats;
int sk_dereplicate(sk_ctx* ctx, const sk_sketch_set* set, const sk_map_params* mp, const uint32_t* rank, const sk_derep_params* dp,
                   uint32_t* rep, uint32_t* cluster, sk_ani_result* join, sk_derep_stats* stats /* may be NULL */);

/* sk_dereplicate_store: sk_dereplicate over every genome of a host sketch store, beyond one GPU's memory and on several GPUs.
 * Contract: for any store (with its name ranks), mp, rank permutation, min_ani, dp->wave, device_budget and context list,
 * rep, cluster and join are byte for byte what sk_dereplicate returns on one in-memory set holding every genome of the store
 * with the same name ranks (join holds store genome ids), and so sk_cluster's greedy result on sk_triangle_store's rows; in
 * stats, pairs_screened, pairs_chained, n_edges, n_clusters, waves and rounds are equal too.
 * The markers of every genome are gathered on ctxs[0] (SK_PACK_MARKERS_ONLY), where the waves, the representative index, the
 * screens and the greedy decisions run exactly as in sk_dereplicate.  Each chain step (a wave against the representatives,
 * the pairs inside a wave, the final members x representatives) is planned into working sets as sk_triangle_store plans
 * its pairs, and the contexts, on one device or several, gather and chain them; every pair is chained once, as
 * (min << 32 | max), in a working set of ascending genome ids, and a gathered set chains exactly like the set that was added.
 * device_budget: bytes per context (0 = derived from the free device memory after the marker gather, ctxs[0]'s device first
 * keeping room for the representative index with every genome a representative).  A genome over budget / 2 gives SK_ERR_NOMEM
 * (before any device work when device_budget is given).  The markers of all genomes stay on ctxs[0]'s device for the whole
 * call (8 bytes per marker).
 * Refusals (SK_ERR_PARAM with the message on ctxs[0]): sk_dereplicate's, plus n_ctx = 0, a NULL context and a context listed
 * twice (n_ctx = 0 or a NULL ctxs / ctxs[0] gives SK_ERR_PARAM without a message).  If any context fails the call fails and
 * sk_last_error(ctxs[0]) carries that context's message.  Stores of 0 and 1 genomes are valid.  SK_TRACE=1 prints one line
 * per working set.
 * stats (may be NULL): as sk_dereplicate's, t_chain covering gathers and chaining (wall time) and t_total the marker gather
 * too.  store_stats (may be NULL): working sets, split components and gathered bytes summed over the chain steps, the largest
 * working set, t_gather / t_chain summed over contexts, t_screen = the marker gather. */
int sk_dereplicate_store(sk_ctx* const* ctxs, uint32_t n_ctx, const sk_sketch_store* st, const sk_map_params* mp, const uint32_t* rank,
                         const sk_derep_params* dp, uint64_t device_budget, uint32_t* rep, uint32_t* cluster, sk_ani_result* join,
                         sk_derep_stats* stats /* may be NULL */, sk_store_stats* store_stats /* may be NULL */);

/* sk_dereplicate_fixed / sk_dereplicate_store_fixed: dereplication that adds genomes to an existing set of representatives.
 * F = { g : rank[g] < n_fixed } are fixed representatives (an earlier run's representatives, a curated catalogue).
 * Contract: rep, cluster and join are what sk_cluster (greedy, same min_ani and rank) returns on the rows of
 * sk_screen_triangle + sk_chain_pairs over the same set and name ranks after every row whose two genomes are both in F is
 * removed; join[g] of a member is byte for byte the row sk_cluster's edge[g] points to, a representative's join is as in
 * sk_dereplicate.  So every genome of F is a representative, even when two of them are joined by an edge; F takes cluster
 * ids 0 .. n_fixed - 1 in rank order and the new clusters follow.  When no two genomes of F share an edge (always the case
 * when F is the representative set of an earlier run at the same threshold and parameters) the result is
 * sk_dereplicate(set, rank)'s.  n_fixed = 0 is sk_dereplicate (sk_dereplicate_store) exactly: outputs, stats and launches.
 * Algorithm: before the first wave F's states are set to representative and its markers form the representative index;
 * the waves cover ranks n_fixed .. N - 1, their wave-size schedule starting at the first genome outside F.  Each wave and the
 * final members x representatives screen run as in sk_dereplicate, F being part of the index from the start.  No pair inside
 * F is ever screened or chained: pairs_screened and pairs_chained count only pairs with a genome outside F, and waves only
 * the waves of genomes outside F (n_fixed = N: no wave, no pair).
 * The result does not depend on dp->wave, device_budget or the context list; the store call equals the in-memory call on one
 * set holding every genome of the store with the same name ranks, stats counts included, as sk_dereplicate_store does.
 * Refusals (SK_ERR_PARAM with a message): n_fixed > n_genomes, plus sk_dereplicate's / sk_dereplicate_store's.  The index
 * limits include F: at most 2^22 - 1 representatives (fixed plus new) and fewer than 2^31 markers in the index; when F
 * alone is over a limit the message names the fixed representatives. */
int sk_dereplicate_fixed(sk_ctx* ctx, const sk_sketch_set* set, const sk_map_params* mp, const uint32_t* rank, uint32_t n_fixed,
                         const sk_derep_params* dp, uint32_t* rep, uint32_t* cluster, sk_ani_result* join,
                         sk_derep_stats* stats /* may be NULL */);
int sk_dereplicate_store_fixed(sk_ctx* const* ctxs, uint32_t n_ctx, const sk_sketch_store* st, const sk_map_params* mp,
                               const uint32_t* rank, uint32_t n_fixed, const sk_derep_params* dp, uint64_t device_budget,
                               uint32_t* rep, uint32_t* cluster, sk_ani_result* join, sk_derep_stats* stats /* may be NULL */,
                               sk_store_stats* store_stats /* may be NULL */);

#ifdef __cplusplus
}
#endif
#endif /* SKANI_B200_H */
