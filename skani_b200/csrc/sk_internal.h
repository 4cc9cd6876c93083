// sk_internal.h -- host-side structures shared by the translation units of libskani_b200.so
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include <atomic>
#include <condition_variable>
#include <functional>
#include <map>
#include <mutex>
#include <string>
#include <thread>
#include <vector>

#include "../../include/skani_b200.h"

// Context-owned device arena: every sketch-set array and every temporary of this library is sub-allocated from a few
// large cudaMalloc'd slabs with host-side first-fit bookkeeping.  All users run on the context's single stream, so a
// block may be handed out again as soon as the host has released it (stream order serialises the accesses).  This keeps
// the steady state free of driver allocation calls: cudaMallocAsync's pool showed multi-100 ms stalls when multi-GB
// blocks of changing size were recycled.
struct SkArena {
  struct Slab { uint8_t* base; size_t size; std::map<size_t, size_t> free_blocks; };  // offset -> size
  std::vector<Slab> slabs;
  std::map<void*, std::pair<int, size_t>> live;   // ptr -> (slab, size)
  std::mutex mu;
  size_t total = 0;
  cudaError_t alloc(void** out, size_t bytes);
  void release(void* p);
  void destroy();
};

// Host worker pool of a context (ASCII -> 2-bit packing and staging copies of sk_sketch_batch).  run() is blocking and
// the caller works too; one run() at a time.
struct SkPool {
  std::vector<std::thread> th;
  std::mutex mu;
  std::condition_variable cv, cv_done;
  const std::function<void(size_t)>* fn = nullptr;
  size_t n_tasks = 0, working = 0;
  std::atomic<size_t> next{0};
  uint64_t gen = 0;
  bool stop = false;
  explicit SkPool(int n_threads);
  ~SkPool();
  void run(size_t n, const std::function<void(size_t)>& f);
  int size() const { return (int)th.size() + 1; }
};

struct sk_ctx {
  SkArena arena;
  int device = 0;
  cudaStream_t stream = nullptr;
  cudaStream_t copy_stream = nullptr;
  std::string err;
  uint64_t launches = 0;
  int sm_count = 132;
  // pinned staging buffers for host->device pipelining (sk_sketch_batch)
  uint8_t* pinned[2] = {nullptr, nullptr};
  size_t pinned_bytes = 0;
  cudaEvent_t pinned_free[2] = {nullptr, nullptr};
  cudaEvent_t h2d_done[2] = {nullptr, nullptr};
  uint8_t* dbuf[2] = {nullptr, nullptr};  // device staging double buffer (sk_sketch_batch): ASCII ...
  size_t dbuf_bytes = 0;
  uint64_t* dP[2] = {nullptr, nullptr};   // ... and 2-bit units + N mask of a sub-batch (host-packed contigs land here directly)
  uint32_t* dNM[2] = {nullptr, nullptr};
  size_t dunits = 0;
  uint64_t* hP[2] = {nullptr, nullptr};   // pinned staging of the host-packed share
  uint32_t* hNM[2] = {nullptr, nullptr};
  size_t hunits = 0;
  cudaEvent_t x0[2] = {nullptr, nullptr}, x1[2] = {nullptr, nullptr};   // timing events around a sub-batch's H2D copies
  SkPool* pool = nullptr;
  int cpu_share = 1;                      // contexts of one process sharing the host cores (sk_triangle_multi)
  bool seed_scalar = false;               // seed with the scalar fmh_seeds semantics (src/seeding.rs:225) instead of avx2_fmh_seeds
  double pack_rate = 0, h2d_rate = 0;     // measured: bases/s packed by the pool, bytes/s over PCIe (adapt the host-packed share)
  double last_pack_share = 0;             // share of the bases packed on the host in the last sk_sketch_batch (stats)
  // correction of the packed share found by hill climbing on the measured host-side stage rate (packing threads and DMA engines
  // share the host's memory bandwidth, which the rate-balancing formula does not know about); persists across calls
  double share_bias = 0, share_ref_rate = 0;
  int share_dir = -1, share_samples = 0;
  double share_acc = 0;
  // small host->device parameter uploads go through a pinned, device-mapped ring + a copy kernel on the context's
  // stream instead of the H2D copy engine, which may be busy for tens of ms with bulk sequence uploads
  uint8_t* stage = nullptr;
  size_t stage_cap = 0, stage_pos = 0;
  // pinned landing blocks for small device->host readbacks (a pageable target makes cudaMemcpyAsync block the host):
  // bump-allocated per seeding sub-batch, reset when the sub-batch is done (seeding.cu)
  std::vector<std::pair<uint8_t*, size_t>> mbox_blocks;
  size_t mbox_block = 0, mbox_pos = 0;
  sk_ctx* child = nullptr;               // worker context of the pipelined sk_triangle (second stream + own workspaces)
  // grow-only chaining workspace (chain.cu), kept for the life of the context
  void* chain_scratch = nullptr;
  void (*chain_scratch_free)(void*) = nullptr;
  // optional per-kernel timing (sk_ctx_set_timing): CUDA events on the launch stream around each major kernel
  bool timing = false;
  struct Pending { const char* name; cudaEvent_t e0, e1; };
  std::vector<Pending> pending;
  std::map<std::string, std::pair<double, uint64_t>> timing_acc;  // name -> (total ms, launches)
};

// launch wrapper: counts the launch and, when timing is on, brackets it with events on ctx->stream
#define SK_LAUNCH(ctx, name, ...)                                     \
  do {                                                                \
    sk_ctx::Pending pe__{name, nullptr, nullptr};                     \
    if ((ctx)->timing) {                                              \
      cudaEventCreate(&pe__.e0); cudaEventCreate(&pe__.e1);           \
      cudaEventRecord(pe__.e0, (ctx)->stream);                        \
    }                                                                 \
    __VA_ARGS__;                                                      \
    (ctx)->launches++;                                                \
    if ((ctx)->timing) {                                              \
      cudaEventRecord(pe__.e1, (ctx)->stream);                        \
      (ctx)->pending.push_back(pe__);                                 \
    }                                                                 \
  } while (0)

struct sk_sketch_set {
  sk_ctx* ctx = nullptr;
  sk_sketch_params sp{};
  uint32_t G = 0;
  // ---- host metadata (prefix offsets have G+1 entries)
  std::vector<uint64_t> seed_off, uk_off, mk_off, ctg_off;
  std::vector<uint32_t> ctg_len;     // all contigs, genome-major
  std::vector<uint64_t> total_len;   // per genome (Sketch.total_sequence_length)
  std::vector<uint64_t> name_rank;   // per genome; order of file names (switch_qr tie-break)
  bool ranks_user_set = false;
  // ---- device arrays
  size_t S = 0, U = 0, M = 0, C = 0;
  uint32_t *pv_kmer = nullptr, *pv_pos = nullptr, *pv_cc = nullptr;  // [S] position-ordered view (genome, contig, pos)
  uint16_t* pv_mult = nullptr;                                        // [S] multiplicity of the record's k-mer in its genome (saturating)
  uint32_t *kv_pos = nullptr, *kv_cc = nullptr;                       // [S] k-mer-ordered view (genome, kmer, contig, pos)
  uint32_t* ukmer = nullptr;                                          // [U] distinct k-mers, ascending per genome
  uint32_t* ustart = nullptr;                                         // [U+G] genome g, group u -> ustart[uk_off[g] + g + u] = local start in kv; +1 sentinel per genome
  uint64_t* markers = nullptr;                                        // [M] sorted distinct per genome
  uint32_t* ctg_rec_off = nullptr;                                    // [C+G] genome g, contig j -> ctg_rec_off[ctg_off[g] + g + j] = local first pv record; +1 sentinel
  uint32_t* d_ctg_len = nullptr;                                      // [C]
  unsigned long long* htab = nullptr;                                 // [ht_off[G]] per-genome open-addressing table: kmer<<32 | start<<12 | min(count,4095); 0 = empty
  std::vector<uint64_t> ht_off;                                       // [G+1] table offsets (capacity = power of two, >= 2 * distinct k-mers); capacity 0 => use ubucket search
  // element capacities of the device arrays when the set grows in place (append_sets_inplace); 0 = allocated at exact size
  size_t capS = 0, capU = 0, capUG = 0, capM = 0, capC = 0, capCG = 0, capHT = 0;
  uint32_t* ubucket = nullptr;                                        // [G * (UBUCKETS + 1)] first ukmer index of each top-bits bucket, per genome
};

#define SK_CUDA(call)                                                                         \
  do {                                                                                        \
    cudaError_t e__ = (call);                                                                 \
    if (e__ != cudaSuccess) {                                                                 \
      ctx->err = std::string(#call) + ": " + cudaGetErrorString(e__) + " (" + __FILE__ + ":" + \
                 std::to_string(__LINE__) + ")";                                              \
      return SK_ERR_CUDA;                                                                     \
    }                                                                                         \
  } while (0)

#define SK_TRY(expr)            \
  do {                          \
    int rc__ = (expr);          \
    if (rc__ != SK_OK) return rc__; \
  } while (0)

// temporary device allocation from the context's arena (released at scope exit)
template <typename T>
struct DTmp {
  T* p = nullptr;
  size_t n = 0;
  sk_ctx* c = nullptr;
  DTmp() {}
  DTmp(const DTmp&) = delete;
  DTmp& operator=(const DTmp&) = delete;
  ~DTmp() { release(); }
  cudaError_t alloc(size_t count, sk_ctx* ctx) {
    release();
    c = ctx;
    n = count;
    if (count == 0) count = 1;
    return ctx->arena.alloc((void**)&p, count * sizeof(T));
  }
  void release() {
    if (p) c->arena.release(p);
    p = nullptr;
    n = 0;
  }
};

namespace sk {
constexpr uint32_t UBUCKET_BITS = 12;
constexpr uint32_t UBUCKETS = 1u << UBUCKET_BITS;
// seeding.cu
struct SeedSrc {                 // where a sub-batch's sequence comes from
  const uint8_t* d_ascii = nullptr;  // device ASCII of the contigs [n_packed, n_contigs): contig i at d_ascii + contig_off[i] - ascii_base
  uint64_t ascii_base = 0;
  uint64_t* d_P = nullptr;           // caller-owned unit arrays of the whole sub-batch with the units of the contigs
  uint32_t* d_NM = nullptr;          //   [0, n_packed) already filled (2-bit codes / N mask); null = allocated by the callee
  uint32_t n_packed = 0;
};
int sketch_batch_device(sk_ctx* ctx, const SeedSrc& src, const uint64_t* contig_off, uint32_t n_contigs,
                        const uint32_t* genome_of_contig, uint32_t n_genomes, const sk_sketch_params* sp, sk_sketch_set** out);
int build_views(sk_ctx* ctx, sk_sketch_set* set, uint64_t* d_marker_raw, const uint64_t* raw_mk_off);   // raw_mk_off: host, [G+1]; may still be in flight on ctx->stream (read after the function's first synchronisation)
void free_set_device(sk_sketch_set* s);
void mbox_reset(sk_ctx* ctx);   // forget the pinned read-back blocks handed out so far (no read-back may be in flight)
int build_hash(sk_ctx* ctx, sk_sketch_set* set);
// api.cu
struct HostSeq {                 // host-resident sequence of a sketch batch: ASCII, or 2-bit units (+ optional N mask)
  const uint8_t* ascii = nullptr;    // contig i at ascii + contig_off[i]
  const uint64_t* units = nullptr;   // contig i at units + sum_{j<i} ceil(len_j / 32); base b of a unit in bits 2b..2b+1
  const uint32_t* nmask = nullptr;   // same indexing, bit b = base b is 'N'; null = no 'N' anywhere
};
int sketch_batch_host(sk_ctx* ctx, const HostSeq& seq, const uint64_t* contig_off, uint32_t n_contigs, const uint32_t* genome_of_contig,
                      uint32_t n_genomes, const sk_sketch_params* sp, sk_sketch_set** out,
                      const std::function<int(sk_sketch_set*, uint32_t, uint32_t)>* on_part, size_t subbatch_override);
int sketch_batch_dev_parts(sk_ctx* ctx, const uint8_t* d_bases, const uint64_t* contig_off, uint32_t n_contigs,
                           const uint32_t* genome_of_contig, uint32_t n_genomes, const sk_sketch_params* sp, sk_sketch_set** out,
                           const std::function<int(sk_sketch_set*, uint32_t, uint32_t)>* on_part, size_t subbatch_override);
SkPool* ctx_pool(sk_ctx* ctx);
// grows `*dst` (created on first use, with capacities reserved for the expected totals) by the genomes of `parts` IN PLACE:
// only the new genomes' arrays are copied and only their k-mer tables are built (the pipelined sk_triangle's merged set)
struct SetReserve { uint64_t bases = 0, contigs = 0, genomes = 0; };
int append_sets_inplace(sk_ctx* ctx, sk_sketch_set** dst, const std::vector<sk_sketch_set*>& parts, const SetReserve& hint);
int build_hash_range(sk_ctx* ctx, sk_sketch_set* set, uint32_t g_begin);   // tables of the genomes [g_begin, G) appended to set->htab
int merge_sets(sk_ctx* ctx, const sk_sketch_set* base, const std::vector<sk_sketch_set*>& parts, sk_sketch_set** out);  // (re)builds set->htab from ukmer/ustart; call on every finished set
// screen.cu: incremental triangle screen of a growing set (pipelined sk_triangle)
struct TriScreen;
int tri_screen_create(sk_ctx* ctx, size_t marker_hint, TriScreen** out);
int tri_screen_add(TriScreen* ts, const sk_sketch_set* set, uint32_t g_end, uint32_t row_begin, const sk_map_params* mp, uint64_t** pairs, uint64_t* n);
void tri_screen_free(TriScreen* ts);
bool tri_screen_supports(uint32_t n_genomes, uint64_t n_markers);
// screen.cu / chain.cu
uint64_t count_launch(sk_ctx* ctx, uint64_t n = 1);
cudaError_t h2d_small(sk_ctx* ctx, void* dst, const void* src, size_t bytes);  // api.cu
}  // namespace sk
