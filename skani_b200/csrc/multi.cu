// multi.cu -- `skani triangle` over several GPUs from ONE host process (SURVEY.md section 8e; the reference's pair loop,
// src/triangle.rs:71-105, is a single rayon process).  One host thread per context:
//   1. contiguous genome blocks (balanced by bases); every device runs the pipelined single-GPU triangle on its own block
//      (sk_triangle_local: upload / seed / screen / chain overlapped) and keeps its sketch set;
//   2. the MARKERS of every block are exchanged device-to-device (peer copies over NVLink when the devices differ, plain
//      device copies when contexts share a device) and every device screens the whole triangle -> the same sorted pair
//      list everywhere, from which the pairs that lie inside one block (already chained in step 1) are dropped;
//   3. the remaining cross-block pairs are split over the devices by connected component (skws::partition_pairs, ws_plan.hpp);
//      a device fetches the sketches its share touches as sub-blobs INCLUDING their k-mer hash tables
//      (sk_sketch_set_pack_subset, SK_PACK_TABLES) and chains them (chain_on_working_set, store_ws.hpp).
// The same steps run as one process per GPU over torch.distributed/NCCL in skani_b200/multi_gpu.py (bench.py --gpus N).
// The query x ref calls touch only their own context's memory, so they need neither peer access nor barriers: one host thread
// per context through run_per_context (store_ws.hpp).
#include <algorithm>
#include <condition_variable>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <mutex>
#include <thread>
#include <vector>

#include "sk_internal.h"
#include "store_ws.hpp"

using sk::now_s;
using sk::enable_peer_access;

extern "C" int sk_triangle_local(sk_ctx* ctx, const uint8_t* bases, const uint64_t* contig_off, uint32_t n_contigs,
                                 const uint32_t* genome_of_contig, uint32_t n_genomes, const sk_sketch_params* sp,
                                 const sk_map_params* mp, const uint64_t* name_ranks, sk_ani_result** out, uint64_t* n_out,
                                 sk_triangle_stats* stats, sk_sketch_set** set_out);

namespace {

struct PhaseBarrier {   // all threads meet; a failure reported by any of them makes everybody leave at the same barrier
  std::mutex mu;
  std::condition_variable cv;
  uint32_t n, count = 0;
  uint64_t gen = 0;
  bool failed = false;
  explicit PhaseBarrier(uint32_t n_) : n(n_) {}
  bool sync(bool ok) {
    std::unique_lock<std::mutex> lk(mu);
    if (!ok) failed = true;
    const uint64_t g = gen;
    if (++count == n) { count = 0; gen++; cv.notify_all(); }
    else cv.wait(lk, [&] { return gen != g; });
    return !failed;
  }
};

struct Blob { void* d = nullptr; uint64_t bytes = 0; std::vector<uint64_t> meta; };

// packs the genomes of s (NULL: all of them) with these flags into a blob in the arena of s's context; errors name `who`
int pack_blob(const char* who, const sk_sketch_set* s, const std::vector<uint32_t>* genomes, int flags, Blob& b) {
  sk_ctx* c = s->ctx;
  const uint32_t none = 0;
  const uint32_t* g = genomes ? (genomes->empty() ? &none : genomes->data()) : nullptr;
  const uint32_t n = genomes ? (uint32_t)genomes->size() : 0;
  uint64_t words = 0;
  SK_TRY(sk_sketch_set_subset_blob_size(s, g, n, flags, &b.bytes, &words));
  if (cudaSetDevice(c->device) != cudaSuccess || c->arena.alloc(&b.d, b.bytes) != cudaSuccess) {
    c->err = std::string(who) + ": out of device memory (source)";
    return SK_ERR_NOMEM;
  }
  b.meta.resize(words);
  return sk_sketch_set_pack_subset(s, g, n, flags, b.d, b.meta.data());
}

// copies the blobs (which may lie on other devices) into one buffer on ctx and unpacks them into one set, in list order;
// errors name `who`
int unpack_blobs(const char* who, sk_ctx* ctx, const std::vector<const Blob*>& blobs, sk_sketch_set** out) {
  const size_t n = blobs.size();
  std::vector<uint64_t> offs(n + 1, 0);
  for (size_t r = 0; r < n; r++) offs[r + 1] = offs[r] + sk::al256(blobs[r]->bytes);
  DTmp<uint8_t> all;
  if (all.alloc(std::max<uint64_t>(offs[n], 256), ctx) != cudaSuccess) { ctx->err = std::string(who) + ": out of device memory (destination)"; return SK_ERR_NOMEM; }
  std::vector<const void*> bp(n);
  std::vector<const uint64_t*> mp(n);
  cudaError_t e = cudaSuccess;
  for (size_t r = 0; r < n && e == cudaSuccess; r++) {
    bp[r] = all.p + offs[r];
    mp[r] = blobs[r]->meta.data();
    e = cudaMemcpyAsync(all.p + offs[r], blobs[r]->d, blobs[r]->bytes, cudaMemcpyDefault, ctx->stream);
  }
  if (e == cudaSuccess) e = cudaStreamSynchronize(ctx->stream);
  if (e != cudaSuccess) { ctx->err = std::string(who) + ": " + cudaGetErrorString(e); return SK_ERR_CUDA; }
  return sk_sketch_set_unpack(ctx, (uint32_t)n, bp.data(), mp.data(), out);
}

}  // namespace

extern "C" int sk_triangle_multi(sk_ctx* const* ctxs, uint32_t n_ctx, const uint8_t* bases, const uint64_t* contig_off, uint32_t n_contigs,
                                 const uint32_t* genome_of_contig, uint32_t n_genomes, const sk_sketch_params* sp,
                                 const sk_map_params* mp, const uint64_t* name_ranks, sk_ani_result** out, uint64_t* n_out,
                                 sk_triangle_stats* stats) {
  if (!ctxs || n_ctx == 0 || !ctxs[0] || !out || !n_out || !sp || !mp || !contig_off || (n_contigs && !genome_of_contig)) return SK_ERR_PARAM;
  *out = nullptr; *n_out = 0;
  sk_ctx* ctx = ctxs[0];
  for (uint32_t d = 0; d < n_ctx; d++) if (!ctxs[d]) { ctx->err = "null context"; return SK_ERR_PARAM; }
  const double t_begin = now_s();
  const uint32_t W = std::min<uint32_t>(n_ctx, std::max<uint32_t>(n_genomes, 1));
  if (W == 1) {
    sk_sketch_set* set = nullptr;
    int rc = sk_triangle_local(ctx, bases, contig_off, n_contigs, genome_of_contig, n_genomes, sp, mp, name_ranks, out, n_out, stats, &set);
    if (set) sk_sketch_set_free(set);
    return rc;
  }
  // ---- genome blocks balanced by bases (every block gets at least one genome)
  std::vector<uint64_t> gbytes(n_genomes, 0);
  for (uint32_t i = 0; i < n_contigs; i++) {
    if (genome_of_contig[i] >= n_genomes || (i && genome_of_contig[i] < genome_of_contig[i - 1])) { ctx->err = "genome_of_contig must be non-decreasing and < n_genomes"; return SK_ERR_PARAM; }
    gbytes[genome_of_contig[i]] += contig_off[i + 1] - contig_off[i];
  }
  uint64_t total = 0;
  for (uint64_t b : gbytes) total += b;
  std::vector<uint32_t> gb(W + 1, 0), cb(W + 1, 0);
  {
    uint64_t acc = 0;
    uint32_t d = 1;
    for (uint32_t g = 0; g < n_genomes && d < W; g++) {
      acc += gbytes[g];
      const uint32_t left_blocks = W - d, left_genomes = n_genomes - (g + 1);
      if (acc * W >= total * d || left_genomes <= left_blocks) { gb[d++] = g + 1; }
    }
    while (d < W) { gb[d] = gb[d - 1]; d++; }
    gb[W] = n_genomes;
    for (uint32_t k = 1; k <= W; k++) gb[k] = std::max(gb[k], gb[k - 1]);
  }
  for (uint32_t d = 0; d <= W; d++) cb[d] = (uint32_t)(std::lower_bound(genome_of_contig, genome_of_contig + n_contigs, gb[d]) - genome_of_contig);
  enable_peer_access(ctxs, W);

  PhaseBarrier bar(W);
  std::vector<sk_sketch_set*> local(W, nullptr);
  std::vector<std::vector<sk_ani_result>> results(W);
  std::vector<Blob> mk(W);
  std::vector<std::vector<Blob>> sub(W, std::vector<Blob>(W));     // sub[src][dst]
  std::vector<std::vector<uint64_t>> cross_part(W);                 // cross-block pairs found by each device's share of the screen
  std::vector<int> rcs(W, SK_OK);
  std::vector<uint64_t> screened(W, 0);
  const bool trace = getenv("SK_TRACE") != nullptr;

  auto run = [&](uint32_t d) -> int {
    sk_ctx* c = ctxs[d];
    int rc = cudaSetDevice(c->device) == cudaSuccess ? SK_OK : SK_ERR_CUDA;   // failures travel to the next barrier: nobody waits for a thread that left
    c->cpu_share = (int)W;
    const double t0 = now_s();
    // ---- 1. own block
    if (rc == SK_OK) {
      std::vector<uint32_t> gl(cb[d + 1] - cb[d]);
      for (uint32_t i = cb[d]; i < cb[d + 1]; i++) gl[i - cb[d]] = genome_of_contig[i] - gb[d];
      sk_ani_result* r = nullptr; uint64_t nr = 0;
      sk_triangle_stats st;
      rc = sk_triangle_local(c, bases, contig_off + cb[d], cb[d + 1] - cb[d], gl.data(), gb[d + 1] - gb[d], sp, mp,
                             name_ranks ? name_ranks + gb[d] : nullptr, &r, &nr, &st, &local[d]);
      if (rc == SK_OK) {
        results[d].assign(r, r + nr);
        for (auto& x : results[d]) { x.ref_id += gb[d]; x.query_id += gb[d]; }
        screened[d] += st.n_pairs_screened;
      }
      if (r) sk_free(r);
    }
    const double t1 = now_s();
    // ---- 2. markers of every block -> every device
    if (rc == SK_OK) rc = pack_blob("sk_triangle_multi", local[d], nullptr, SK_PACK_MARKERS_ONLY, mk[d]);
    if (!bar.sync(rc == SK_OK)) return rc;
    sk_sketch_set* mkset = nullptr;
    {
      std::vector<const Blob*> from(W);
      for (uint32_t r = 0; r < W; r++) from[r] = &mk[r];
      rc = unpack_blobs("sk_triangle_multi", c, from, &mkset);
    }
    if (!bar.sync(rc == SK_OK)) { if (mkset) sk_sketch_set_free(mkset); return rc; }   // every peer has copied: the marker blobs may go
    c->arena.release(mk[d].d); mk[d].d = nullptr;
    // ---- sharded screen: this device screens the rows of ITS block against every genome before them (one sort of the markers of
    //      the blocks up to its own, rows of one block) and keeps the pairs that cross a block boundary; the W partial lists are
    //      exchanged through host memory and merged, so that every device holds the same sorted cross-block pair list
    uint64_t* pairs = nullptr; uint64_t np = 0;
    rc = sk_screen_triangle_block(c, mkset, gb[d], gb[d + 1], mp, &pairs, &np);
    sk_sketch_set_free(mkset);
    if (rc == SK_OK) {
      cross_part[d].clear();
      for (uint64_t i = 0; i < np; i++) if ((uint32_t)(pairs[i] >> 32) < gb[d]) cross_part[d].push_back(pairs[i]);
      sk_free(pairs);
    }
    if (!bar.sync(rc == SK_OK)) return rc;
    std::vector<uint64_t> cross;
    for (uint32_t r = 0; r < W; r++) cross.insert(cross.end(), cross_part[r].begin(), cross_part[r].end());
    std::sort(cross.begin(), cross.end());
    const double t2 = now_s();
    // split over the devices by connected component of the pair graph (every thread computes the same split)
    std::vector<std::vector<uint64_t>> share;
    skws::partition_pairs(cross, W, n_genomes, share);
    auto genomes_of_slice = [&](uint32_t r, std::vector<uint32_t>& need) {
      need.clear();
      for (uint64_t pr : share[r]) { need.push_back((uint32_t)(pr >> 32)); need.push_back((uint32_t)pr); }
      std::sort(need.begin(), need.end());
      need.erase(std::unique(need.begin(), need.end()), need.end());
    };
    // ---- 3. pack what every device needs from this block (the pair list is identical everywhere, so no request round)
    std::vector<uint32_t> need, mine;
    for (uint32_t r = 0; r < W && rc == SK_OK; r++) {
      genomes_of_slice(r, need);
      if (r == d) mine = need;
      std::vector<uint32_t> loc;
      for (uint32_t g : need) if (g >= gb[d] && g < gb[d + 1]) loc.push_back(g - gb[d]);
      rc = pack_blob("sk_triangle_multi", local[d], &loc, SK_PACK_TABLES, sub[d][r]);
    }
    if (!bar.sync(rc == SK_OK)) return rc;
    sk_sketch_set* work = nullptr;
    uint64_t remote_bytes = 0;
    {
      std::vector<const Blob*> from(W);
      for (uint32_t r = 0; r < W; r++) {
        from[r] = &sub[r][d];
        if (r != d) remote_bytes += sub[r][d].bytes;
      }
      rc = unpack_blobs("sk_triangle_multi", c, from, &work);     // source-block order = ascending global ids
    }
    if (!bar.sync(rc == SK_OK)) { if (work) sk_sketch_set_free(work); return rc; }     // every peer has copied its sub-blobs
    for (uint32_t r = 0; r < W; r++) if (sub[d][r].d) { c->arena.release(sub[d][r].d); sub[d][r].d = nullptr; }
    sk_sketch_set_free(local[d]); local[d] = nullptr;
    const double t3 = now_s();
    // ---- chain the slice on the working set
    const std::vector<uint64_t>& my_pairs = share[d];
    if (rc == SK_OK && !my_pairs.empty()) {
      if (sk_sketch_set_n_genomes(work) != mine.size()) { c->err = "fetch plan mismatch"; rc = SK_ERR_STATE; }
      std::vector<uint64_t> ranks(mine.size());
      for (size_t i = 0; i < mine.size(); i++) ranks[i] = name_ranks ? name_ranks[mine[i]] : mine[i];
      if (rc == SK_OK) rc = sk_sketch_set_set_name_ranks(work, ranks.data());
      std::vector<sk_ani_result> res;
      if (rc == SK_OK) rc = sk::chain_on_working_set(c, work, mine, work, mine, my_pairs, mp, res);
      if (rc == SK_OK)
        for (const auto& x : res)
          if (x.ani > 0.1f) results[d].push_back(x);   // src/triangle.rs:99
      screened[d] += my_pairs.size();
    }
    if (work) sk_sketch_set_free(work);
    if (trace) fprintf(stderr, "[sk_triangle_multi] device slot %u (gpu %d): block %u..%u local %.1f ms, markers+screen %.1f ms, fetch %.1f ms "
                               "(%zu genomes, %.1f MB remote), chain %.1f ms (%llu cross-block pairs of %zu)\n", d, c->device, gb[d], gb[d + 1],
                       (t1 - t0) * 1e3, (t2 - t1) * 1e3, (t3 - t2) * 1e3, mine.size(), remote_bytes / 1e6, (now_s() - t3) * 1e3,
                       (unsigned long long)my_pairs.size(), cross.size());
    return rc;
  };

  std::vector<std::thread> th;
  for (uint32_t d = 0; d < W; d++)
    th.emplace_back([&, d] {
      rcs[d] = run(d);
    });
  for (auto& t : th) t.join();
  int rc = SK_OK;
  for (uint32_t d = 0; d < W; d++) {
    if (rcs[d] != SK_OK && rc == SK_OK) { rc = rcs[d]; if (d) ctx->err = "device slot " + std::to_string(d) + ": " + ctxs[d]->err; }
    cudaSetDevice(ctxs[d]->device);
    if (local[d]) sk_sketch_set_free(local[d]);
    if (mk[d].d) ctxs[d]->arena.release(mk[d].d);
    for (uint32_t r = 0; r < W; r++) if (sub[d][r].d) ctxs[d]->arena.release(sub[d][r].d);
  }
  cudaSetDevice(ctx->device);
  if (rc != SK_OK) return rc;
  std::vector<sk_ani_result> all;
  for (auto& v : results) all.insert(all.end(), v.begin(), v.end());
  SK_TRY(sk::hand_out(ctx, all, out, n_out));
  if (stats) {
    memset(stats, 0, sizeof(*stats));
    stats->t_total = now_s() - t_begin;
    for (uint64_t s : screened) stats->n_pairs_screened += s;
    stats->n_pairs_kept = all.size();
  }
  return SK_OK;
}

// ---- query x ref work over several contexts (`skani dist` / `skani search` with --gpus N, src/dist.rs:98-144,
//      src/search.rs:119-247).  The references are split into contiguous blocks, one per context; the query set is copied
//      to every context.  A (ref, query) pair's screen decision and chain result depend on that pair alone, so each context
//      screens / chains its own block and the per-block results are put back in the caller's order with global ref ids.

extern "C" int sk_sketch_set_copy(sk_ctx* dst, const sk_sketch_set* src, sk_sketch_set** out) {
  if (!dst || !src || !out) return SK_ERR_PARAM;
  *out = nullptr;
  sk_ctx* sc = src->ctx;
  if (dst != sc) { sk_ctx* pair[2] = {sc, dst}; enable_peer_access(pair, 2); }
  // the source set's own blob, k-mer tables included (no rebuild on the destination), copied device to device
  Blob blob;
  int rc = pack_blob("sk_sketch_set_copy", src, nullptr, SK_PACK_TABLES, blob);   // synchronises the source stream
  if (rc == SK_OK && dst == sc) {
    const void* bp = blob.d;
    const uint64_t* mp = blob.meta.data();
    rc = sk_sketch_set_unpack(dst, 1, &bp, &mp, out);
  } else if (rc == SK_OK) {
    const cudaError_t e = cudaSetDevice(dst->device);
    if (e == cudaSuccess) rc = unpack_blobs("sk_sketch_set_copy", dst, {&blob}, out);
    else { dst->err = std::string("sk_sketch_set_copy: ") + cudaGetErrorString(e); rc = SK_ERR_CUDA; }
  } else if (dst != sc) {
    dst->err = sc->err;
  }
  if (rc == SK_OK) { (*out)->name_rank = src->name_rank; (*out)->ranks_user_set = src->ranks_user_set; }   // host-side state
  if (blob.d) { cudaSetDevice(sc->device); sc->arena.release(blob.d); }
  cudaSetDevice(dst->device);
  return rc;
}

namespace {

struct QrBlocks {
  std::vector<uint32_t> G;   // references held by each context (0 for a NULL set)
  uint64_t n_refs = 0;       // end of the last block: the size of the one set the blocks stand for
  uint32_t n_queries = 0;
};

// the arguments shared by the two query x ref calls; every violation is the caller's and is reported on ctxs[0]
int check_qr_args(sk_ctx* const* ctxs, uint32_t n_ctx, const sk_sketch_set* const* refs, const uint32_t* ref_first,
                  const sk_sketch_set* const* queries, const sk_map_params* mp, QrBlocks& qb) {
  if (!ctxs || n_ctx == 0 || !ctxs[0]) return SK_ERR_PARAM;
  sk_ctx* ctx = ctxs[0];
  auto fail = [&](const std::string& m) { ctx->err = m; return SK_ERR_PARAM; };
  if (!refs || !ref_first || !queries || !mp) return fail("NULL argument");
  if (!queries[0]) return fail("queries[0] is NULL");
  SK_TRY(sk::check_contexts(ctxs, n_ctx));
  const sk_sketch_set* q0 = queries[0];
  qb.G.assign(n_ctx, 0);
  for (uint32_t d = 0; d < n_ctx; d++) {
    const std::string at = "context " + std::to_string(d) + ": ";
    const sk_sketch_set* q = queries[d];
    if (!q || q->ctx != ctxs[d]) return fail(at + "queries[d] must be a set of ctxs[d]");
    if (q->G != q0->G || q->seed_off != q0->seed_off || q->mk_off != q0->mk_off || q->ctg_off != q0->ctg_off)
      return fail(at + "queries[d] is not the query set of context 0 (copy it with sk_sketch_set_copy)");
    if (!sk::same_params(q->sp, q0->sp)) return fail(at + "sketch parameters differ");
    if (refs[d]) {
      if (refs[d]->ctx != ctxs[d]) return fail(at + "refs[d] must be a set of ctxs[d]");
      if (!sk::same_params(refs[d]->sp, q0->sp)) return fail(at + "sketch parameters differ");
      qb.G[d] = refs[d]->G;
    }
    if (d && (uint64_t)ref_first[d] < (uint64_t)ref_first[d - 1] + qb.G[d - 1]) return fail(at + "ref_first must be ascending and the blocks disjoint");
    if ((uint64_t)ref_first[d] + qb.G[d] > (1ull << 32)) return fail(at + "global ref ids must fit 32 bits");
  }
  qb.n_refs = (uint64_t)ref_first[n_ctx - 1] + qb.G[n_ctx - 1];
  qb.n_queries = q0->G;
  return SK_OK;
}

}  // namespace

extern "C" int sk_screen_query_ref_multi(sk_ctx* const* ctxs, uint32_t n_ctx, const sk_sketch_set* const* refs, const uint32_t* ref_first,
                                         const sk_sketch_set* const* queries, const sk_map_params* mp, int mode,
                                         uint64_t** pairs_rq, uint64_t* n_pairs) {
  if (!pairs_rq || !n_pairs) return SK_ERR_PARAM;
  *pairs_rq = nullptr; *n_pairs = 0;
  QrBlocks qb;
  SK_TRY(check_qr_args(ctxs, n_ctx, refs, ref_first, queries, mp, qb));
  if (mode < 0 || mode > 3) { ctxs[0]->err = "mode must be 0..3"; return SK_ERR_PARAM; }
  std::vector<std::vector<uint64_t>> part(n_ctx);
  SK_TRY(sk::run_per_context(ctxs, n_ctx, [&](uint32_t d) -> int {
    if (qb.G[d] == 0) return SK_OK;
    uint64_t* p = nullptr; uint64_t n = 0;
    const int rc = sk_screen_query_ref(ctxs[d], refs[d], queries[d], mp, mode, &p, &n);
    if (rc == SK_OK) {
      const uint64_t shift = (uint64_t)ref_first[d] << 32;     // (local ref << 32 | query) -> global ref
      part[d].resize(n);
      for (uint64_t i = 0; i < n; i++) part[d][i] = p[i] + shift;
    }
    if (p) sk_free(p);
    return rc;
  }));
  // every block's list is sorted and the blocks ascend: their concatenation is sorted
  std::vector<uint64_t> all;
  for (auto& v : part) all.insert(all.end(), v.begin(), v.end());
  return sk::hand_out(ctxs[0], all, pairs_rq, n_pairs);
}

// sk_chain_pairs_multi, and with map_off / maps non-null sk_chain_pairs_multi_mappings
static int chain_pairs_multi(sk_ctx* const* ctxs, uint32_t n_ctx, const sk_sketch_set* const* refs, const uint32_t* ref_first,
                             const sk_sketch_set* const* queries, const uint64_t* pairs, uint64_t n_pairs,
                             const sk_map_params* mp, sk_ani_result* out, uint64_t* map_off, sk_mapping** maps) {
  QrBlocks qb;
  SK_TRY(check_qr_args(ctxs, n_ctx, refs, ref_first, queries, mp, qb));
  if (n_pairs && (!pairs || !out)) { ctxs[0]->err = "NULL pairs / out"; return SK_ERR_PARAM; }
  // route every pair to the block holding its ref (pairs may come in any order)
  std::vector<std::vector<uint64_t>> local(n_ctx);
  std::vector<std::vector<uint64_t>> where(n_ctx);      // index of the pair in the caller's list
  for (uint64_t i = 0; i < n_pairs; i++) {
    const uint32_t r = (uint32_t)(pairs[i] >> 32), q = (uint32_t)pairs[i];
    if (q >= qb.n_queries) { ctxs[0]->err = "pair " + std::to_string(i) + ": query index out of range"; return SK_ERR_PARAM; }
    const uint32_t* it = std::upper_bound(ref_first, ref_first + n_ctx, r);
    const uint32_t d = (uint32_t)(it - ref_first) - 1;
    if (it == ref_first || r - ref_first[d] >= qb.G[d]) { ctxs[0]->err = "pair " + std::to_string(i) + ": ref " + std::to_string(r) + " lies in no block"; return SK_ERR_PARAM; }
    local[d].push_back(((uint64_t)(r - ref_first[d]) << 32) | q);
    where[d].push_back(i);
  }
  const bool with_maps = map_off != nullptr;
  std::vector<std::vector<uint64_t>> loff(n_ctx);       // mappings: each context's offsets and records, in its local order
  std::vector<sk_mapping*> lmaps(n_ctx, nullptr);
  const int rc = sk::run_per_context(ctxs, n_ctx, [&](uint32_t d) -> int {
    if (local[d].empty()) return SK_OK;
    // switch_qr's file-name tie-break (src/chain.rs:19-21) as in the one set of all refs: default ranks are global ref ids,
    // and default query ranks follow all n_refs refs.  Applied on non-owning views; the caller's sets are not touched.
    sk_sketch_set rv = *refs[d], qv = *queries[d];
    if (!rv.ranks_user_set) for (uint32_t g = 0; g < rv.G; g++) rv.name_rank[g] = (uint64_t)ref_first[d] + g;
    if (!qv.ranks_user_set) for (uint32_t g = 0; g < qv.G; g++) qv.name_rank[g] += qb.n_refs;
    rv.ranks_user_set = qv.ranks_user_set = true;
    std::vector<sk_ani_result> res(local[d].size());
    int rc;
    if (with_maps) {
      loff[d].resize(local[d].size() + 1);
      rc = sk_chain_pairs_mappings(ctxs[d], &rv, &qv, local[d].data(), local[d].size(), mp, res.data(), loff[d].data(), &lmaps[d]);
    } else {
      rc = sk_chain_pairs(ctxs[d], &rv, &qv, local[d].data(), local[d].size(), mp, res.data());
    }
    if (rc != SK_OK) return rc;
    for (size_t k = 0; k < res.size(); k++) { res[k].ref_id += ref_first[d]; out[where[d][k]] = res[k]; }
    return SK_OK;
  });
  if (rc == SK_OK && with_maps) {
    // records merged back into the caller's pair order
    std::vector<uint32_t> ctx_of(n_pairs);
    std::vector<uint64_t> k_of(n_pairs);
    for (uint32_t d = 0; d < n_ctx; d++)
      for (size_t k = 0; k < where[d].size(); k++) { ctx_of[where[d][k]] = d; k_of[where[d][k]] = k; }
    map_off[0] = 0;
    for (uint64_t i = 0; i < n_pairs; i++) map_off[i + 1] = map_off[i] + loff[ctx_of[i]][k_of[i] + 1] - loff[ctx_of[i]][k_of[i]];
    *maps = (sk_mapping*)malloc(std::max<uint64_t>(map_off[n_pairs], 1) * sizeof(sk_mapping));
    if (*maps)
      for (uint64_t i = 0; i < n_pairs; i++) {
        const uint64_t* lo = loff[ctx_of[i]].data() + k_of[i];
        if (lo[1] > lo[0]) memcpy(*maps + map_off[i], lmaps[ctx_of[i]] + lo[0], (lo[1] - lo[0]) * sizeof(sk_mapping));
      }
  }
  for (sk_mapping* m : lmaps) sk_free(m);
  if (rc == SK_OK && with_maps && !*maps) { ctxs[0]->err = "chain mappings: out of host memory"; return SK_ERR_NOMEM; }
  return rc;
}

extern "C" int sk_chain_pairs_multi(sk_ctx* const* ctxs, uint32_t n_ctx, const sk_sketch_set* const* refs, const uint32_t* ref_first,
                                    const sk_sketch_set* const* queries, const uint64_t* pairs, uint64_t n_pairs,
                                    const sk_map_params* mp, sk_ani_result* out) {
  return chain_pairs_multi(ctxs, n_ctx, refs, ref_first, queries, pairs, n_pairs, mp, out, nullptr, nullptr);
}

extern "C" int sk_chain_pairs_multi_mappings(sk_ctx* const* ctxs, uint32_t n_ctx, const sk_sketch_set* const* refs,
                                             const uint32_t* ref_first, const sk_sketch_set* const* queries, const uint64_t* pairs,
                                             uint64_t n_pairs, const sk_map_params* mp, sk_ani_result* out, uint64_t* map_off,
                                             sk_mapping** maps) {
  if (!map_off || !maps) return SK_ERR_PARAM;
  *maps = nullptr;
  return chain_pairs_multi(ctxs, n_ctx, refs, ref_first, queries, pairs, n_pairs, mp, out, map_off, maps);
}
