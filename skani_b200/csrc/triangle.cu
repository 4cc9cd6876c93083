// triangle.cu -- whole `skani triangle` hot path from host buffers (reference src/triangle.rs:13-105):
// sketch every genome, marker screen (rows i, columns j > i), chain every passing pair, keep ani > 0.1.
//
// Large inputs are PCIe-bound (a 5 Mbp genome is 5 MB of ASCII on the wire and ~70 us of kernels), so the call is
// software-pipelined: the genome set is cut into waves; while wave w+1 is being uploaded and seeded on the context's
// stream, a worker thread with a child context appends wave w to the set sketched so far, screens it and chains the
// NEW pairs (those whose larger index lies in wave w) on a second stream.  The result set is identical to the
// unpipelined order of operations: pair (i, j), i < j, is screened by row i's rule against all columns exactly once,
// when j's wave arrives (src/triangle.rs:71-105 evaluates the same predicate on the same sketches).
#include <chrono>
#include <condition_variable>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <algorithm>
#include <deque>
#include <functional>
#include <mutex>
#include <thread>
#include <vector>

#include "sk_internal.h"

extern "C" int sk_ctx_create_worker(int device, sk_ctx** out);   // api.cu: a context whose stream has the LOWEST priority

namespace {

struct Wave { sk_sketch_set* set; uint32_t g_begin; bool last; };

bool is_device_ptr(const void* p) {
  if (!p) return false;
  cudaPointerAttributes attr;
  const bool dev = cudaPointerGetAttributes(&attr, p) == cudaSuccess && attr.type == cudaMemoryTypeDevice;
  cudaGetLastError();
  return dev;
}

double now_s() { return std::chrono::duration<double>(std::chrono::steady_clock::now().time_since_epoch()).count(); }

int simple_triangle(sk_ctx* ctx, const sk::HostSeq& seq, const uint64_t* contig_off, uint32_t n_contigs, const uint32_t* genome_of_contig,
                    uint32_t n_genomes, const sk_sketch_params* sp, const sk_map_params* mp, std::vector<sk_ani_result>& kept,
                    uint64_t* n_screened, sk_sketch_set** keep, const uint64_t* name_ranks) {
  sk_sketch_set* set = nullptr;
  if (seq.units && n_contigs && contig_off[n_contigs] > contig_off[0]) SK_TRY(sk::sketch_batch_host(ctx, seq, contig_off, n_contigs, genome_of_contig, n_genomes, sp, &set, nullptr, 0));
  else if (is_device_ptr(seq.ascii)) SK_TRY(sk_sketch_batch_dev(ctx, seq.ascii, contig_off, n_contigs, genome_of_contig, n_genomes, sp, &set));
  else SK_TRY(sk_sketch_batch(ctx, seq.ascii ? seq.ascii : (const uint8_t*)"", contig_off, n_contigs, genome_of_contig, n_genomes, sp, &set));
  if (name_ranks) sk_sketch_set_set_name_ranks(set, name_ranks);
  struct SG { sk_sketch_set* s; sk_sketch_set** keep; ~SG() { if (keep && s) *keep = s; else sk_sketch_set_free(s); } } sg{set, keep};
  if (keep) *keep = nullptr;
  uint64_t* pairs = nullptr;
  uint64_t np = 0;
  SK_TRY(sk_screen_triangle(ctx, set, mp, &pairs, &np));
  struct PG { uint64_t* p; ~PG() { free(p); } } pg{pairs};
  std::vector<sk_ani_result> res(np);
  SK_TRY(sk_chain_pairs(ctx, set, set, pairs, np, mp, res.data()));
  for (auto& r : res) if (r.ani > 0.1f) kept.push_back(r);            // src/triangle.rs:99 (NaN and -1 fail)
  *n_screened = np;
  return SK_OK;
}

int triangle_impl(sk_ctx* ctx, const sk::HostSeq& seq, const uint64_t* contig_off, uint32_t n_contigs,
                  const uint32_t* genome_of_contig, uint32_t n_genomes, const sk_sketch_params* sp,
                  const sk_map_params* mp, sk_ani_result** out, uint64_t* n_out, sk_triangle_stats* stats, sk_sketch_set** keep,
                  const uint64_t* name_ranks);

}  // namespace

extern "C" int sk_triangle(sk_ctx* ctx, const uint8_t* bases, const uint64_t* contig_off, uint32_t n_contigs,
                           const uint32_t* genome_of_contig, uint32_t n_genomes, const sk_sketch_params* sp,
                           const sk_map_params* mp, sk_ani_result** out, uint64_t* n_out, sk_triangle_stats* stats) {
  sk::HostSeq seq; seq.ascii = bases;
  return triangle_impl(ctx, seq, contig_off, n_contigs, genome_of_contig, n_genomes, sp, mp, out, n_out, stats, nullptr, nullptr);
}

extern "C" int sk_triangle_local(sk_ctx* ctx, const uint8_t* bases, const uint64_t* contig_off, uint32_t n_contigs,
                                 const uint32_t* genome_of_contig, uint32_t n_genomes, const sk_sketch_params* sp,
                                 const sk_map_params* mp, const uint64_t* name_ranks, sk_ani_result** out, uint64_t* n_out,
                                 sk_triangle_stats* stats, sk_sketch_set** set_out) {
  if (!set_out) return SK_ERR_PARAM;
  sk::HostSeq seq; seq.ascii = bases;
  return triangle_impl(ctx, seq, contig_off, n_contigs, genome_of_contig, n_genomes, sp, mp, out, n_out, stats, set_out, name_ranks);
}

// the same for callers that hold their genomes 2-bit packed (sk_sketch_batch_2bit's layout): 0.25 B/base leave host memory
extern "C" int sk_triangle_2bit(sk_ctx* ctx, const uint64_t* units, const uint32_t* nmask, const uint32_t* contig_len, uint32_t n_contigs,
                                const uint32_t* genome_of_contig, uint32_t n_genomes, const sk_sketch_params* sp,
                                const sk_map_params* mp, const uint64_t* name_ranks, sk_ani_result** out, uint64_t* n_out,
                                sk_triangle_stats* stats, sk_sketch_set** set_out) {
  if (!ctx || (n_contigs && (!units || !contig_len || !genome_of_contig))) return SK_ERR_PARAM;
  std::vector<uint64_t> off((size_t)n_contigs + 1, 0);
  for (uint32_t i = 0; i < n_contigs; i++) off[i + 1] = off[i] + contig_len[i];
  sk::HostSeq seq; seq.units = units; seq.nmask = nmask;
  return triangle_impl(ctx, seq, off.data(), n_contigs, genome_of_contig, n_genomes, sp, mp, out, n_out, stats, set_out, name_ranks);
}

namespace {
int triangle_impl(sk_ctx* ctx, const sk::HostSeq& seq, const uint64_t* contig_off, uint32_t n_contigs,
                  const uint32_t* genome_of_contig, uint32_t n_genomes, const sk_sketch_params* sp,
                  const sk_map_params* mp, sk_ani_result** out, uint64_t* n_out, sk_triangle_stats* stats, sk_sketch_set** keep,
                  const uint64_t* name_ranks) {
  if (!ctx || !out || !n_out || !sp || !mp || !contig_off) return SK_ERR_PARAM;
  *out = nullptr; *n_out = 0;
  if (keep) *keep = nullptr;
  SK_CUDA(cudaSetDevice(ctx->device));
  cudaEvent_t ev[2];
  for (auto& e : ev) SK_CUDA(cudaEventCreate(&e));
  struct EG { cudaEvent_t* e; ~EG() { for (int i = 0; i < 2; i++) cudaEventDestroy(e[i]); } } eg{ev};
  SK_CUDA(cudaEventRecord(ev[0], ctx->stream));
  std::vector<sk_ani_result> kept;
  uint64_t n_screened = 0;
  const uint64_t total_bytes = n_contigs ? contig_off[n_contigs] - contig_off[0] : 0;
  // Inputs of >= 4 GiB use the upload/seed || merge/screen/chain pipeline (SK_NO_PIPELINE=1 disables it, SK_FORCE_PIPELINE=1
  // forces it for small inputs in tests).  Two things made it work: the context arena (no driver allocations in steady
  // state) and h2d_small (parameter uploads bypass the H2D copy engine that is saturated by the sequence upload).
  // memory guard: the whole sketch set stays resident (records 22 B + k-mer tables <= 32 B per seed, markers 8 B each, plus the
  // chaining workspace); refuse up front instead of failing half-way through a long run -- more genomes than one GPU holds
  // go through sk_triangle_multi (blocks per GPU), SURVEY.md section 8 config 4
  {
    size_t free_b = 0, total_b = 0;
    if (cudaMemGetInfo(&free_b, &total_b) == cudaSuccess) {
      const double need = (double)total_bytes / sp->c * 56.0 + (double)total_bytes / sp->marker_c * 24.0 + 6.0e9;
      if (need > 0.92 * (double)total_b) {
        ctx->err = "input too large for one GPU: ~" + std::to_string((uint64_t)(need / 1e9)) + " GB of sketches + workspace vs " +
                   std::to_string((uint64_t)(total_b / 1e9)) + " GB of device memory; use sk_triangle_multi (triangle --gpus N)";
        return SK_ERR_NOMEM;
      }
    }
  }
  const bool pipelined = ((total_bytes >= (4ull << 30) && n_genomes >= 64) || (getenv("SK_FORCE_PIPELINE") && n_genomes >= 2)) &&
                         getenv("SK_NO_PIPELINE") == nullptr && n_contigs > 0;
  if (!pipelined) {
    int rc = simple_triangle(ctx, seq, contig_off, n_contigs, genome_of_contig, n_genomes, sp, mp, kept, &n_screened, keep, name_ranks);
    if (rc != SK_OK) { if (keep && *keep) { sk_sketch_set_free(*keep); *keep = nullptr; } return rc; }
  } else {
    // ---- producer: ONE continuous upload + seeding pass (the H2D stream never drains); every finished sub-batch is
    //      handed to the worker.  Worker: once >= 1/8 of the genomes are pending (or the input is finished) it merges
    //      them into the set sketched so far, screens the merged set and chains the pairs whose larger index is new.
    if (!ctx->child) {
      if (sk_ctx_create_worker(ctx->device, &ctx->child) != SK_OK) { ctx->err = "cannot create the worker context"; return SK_ERR_CUDA; }
      ctx->child->seed_scalar = ctx->seed_scalar;
    }
    sk_ctx* wctx = ctx->child;
    const bool trace = getenv("SK_TRACE") != nullptr;
    const double t00 = now_s();
    const uint32_t wave_genomes = std::max<uint32_t>(1, n_genomes / 8);
    sk::SetReserve reserve;
    reserve.bases = total_bytes; reserve.contigs = n_contigs; reserve.genomes = n_genomes;
    std::mutex mu;
    std::condition_variable cv;
    std::deque<Wave> q;
    int worker_rc = SK_OK;
    std::string worker_err;
    sk_sketch_set* merged = nullptr;        // the set sketched so far (owned by the worker context's arena)
    // incremental screen: the sorted marker table of the merged set is kept and each wave only adds its own markers and
    // screens its own genomes (SK_FULL_RESCREEN=1: screen the whole merged set every wave and filter, as round 1 did)
    sk::TriScreen* tscreen = nullptr;
    const bool inc_screen = getenv("SK_FULL_RESCREEN") == nullptr &&
                            sk::tri_screen_supports(n_genomes, (uint64_t)((double)total_bytes / sp->marker_c * 1.5) + n_genomes);
    std::thread worker([&] {
      cudaSetDevice(wctx->device);
      std::vector<sk_sketch_set*> pending;
      uint32_t pending_begin = 0, pending_genomes = 0;
      bool done = false;
      while (!done) {
        Wave w;
        {
          std::unique_lock<std::mutex> lk(mu);
          cv.wait(lk, [&] { return !q.empty(); });
          w = q.front(); q.pop_front();
        }
        if (w.set) {
          if (pending.empty()) pending_begin = w.g_begin;
          pending.push_back(w.set);
          pending_genomes += w.set->G;
        }
        done = w.last;
        // wave size: n/8 while plenty is still to come, then half of what is left (down to n/64), so that the work that
        // remains after the LAST upload -- one screen + the chains of the last wave -- is small (the pipeline's tail)
        const uint32_t merged_g = merged ? merged->G : 0;
        const uint32_t left = n_genomes - std::min(n_genomes, merged_g);          // genomes not merged yet (pending included)
        const uint32_t threshold = std::max<uint32_t>(std::max<uint32_t>(1, n_genomes / 64), std::min(wave_genomes, left / 2));
        if (pending.empty() || (!done && pending_genomes < threshold)) continue;
        if (worker_rc == SK_OK) {
          const double ta = now_s();
          // the merged set grows in place: only the new genomes are copied and only their k-mer tables are built
          int rc = sk::append_sets_inplace(wctx, &merged, pending, reserve);
          double tb = now_s(), tc = tb, td = tb;
          if (rc == SK_OK) {
            if (name_ranks) {   // file-name order of the caller (switch_qr tie-break); the merged set covers genomes [0, merged->G)
              for (uint32_t g = 0; g < merged->G; g++) merged->name_rank[g] = name_ranks[g];
              merged->ranks_user_set = true;
            }
            uint64_t* pairs = nullptr; uint64_t np = 0;
            bool inc = inc_screen && sk::tri_screen_supports(merged->G, merged->M);
            if (inc && !tscreen) rc = sk::tri_screen_create(wctx, (size_t)((double)total_bytes / sp->marker_c * 1.1) + 1024, &tscreen);
            if (rc == SK_OK) rc = inc ? sk::tri_screen_add(tscreen, merged, merged->G, pending_begin, mp, &pairs, &np)
                                      : sk_screen_triangle(wctx, merged, mp, &pairs, &np);
            tc = now_s();
            if (rc == SK_OK) {
              uint64_t m = 0;   // new pairs: larger index j inside the genomes just merged
              for (uint64_t i = 0; i < np; i++) if ((uint32_t)pairs[i] >= pending_begin) pairs[m++] = pairs[i];
              std::vector<sk_ani_result> res(m);
              rc = sk_chain_pairs(wctx, merged, merged, pairs, m, mp, res.data());
              if (rc == SK_OK) { for (auto& r : res) if (r.ani > 0.1f) kept.push_back(r); n_screened += m; }
              free(pairs);
              td = now_s();
            }
          }
          if (trace) fprintf(stderr, "[sk_triangle] worker: genomes >= %u (%u new): start %.3f merge %.3f screen %.3f chain %.3f s\n",
                             pending_begin, pending_genomes, ta - t00, tb - ta, tc - tb, td - tc);
          if (rc != SK_OK) { worker_rc = rc; worker_err = wctx->err; }
        }
        cudaStreamSynchronize(wctx->stream);
        for (auto* p : pending) sk_sketch_set_free(p);
        pending.clear(); pending_genomes = 0;
      }
      cudaStreamSynchronize(wctx->stream);
      sk::tri_screen_free(tscreen);
    });
    std::function<int(sk_sketch_set*, uint32_t, uint32_t)> on_part = [&](sk_sketch_set* part, uint32_t g_begin, uint32_t g_end) -> int {
      (void)g_end;
      if (trace) fprintf(stderr, "[sk_triangle] producer: part of %u genomes from %u ready at %.3f s\n", part->G, g_begin, now_s() - t00);
      { std::lock_guard<std::mutex> lk(mu); q.push_back(Wave{part, g_begin, false}); }
      cv.notify_one();
      return SK_OK;
    };
    // sub-batches of 1 .. 2 GiB (about 1/16 of the input): 2 GiB measured 10 % faster end to end than 1 GiB on the 50 GB run
    const size_t subbatch = (size_t)std::min<uint64_t>(2048ull << 20, std::max<uint64_t>(1024ull << 20, total_bytes / 16));
    // genomes already resident on the device (bases = device pointer): the same pipeline without the pack / upload stages
    const bool dev_src = is_device_ptr(seq.ascii);
    int rc = dev_src ? sk::sketch_batch_dev_parts(ctx, seq.ascii, contig_off, n_contigs, genome_of_contig, n_genomes, sp, nullptr, &on_part, subbatch)
                     : sk::sketch_batch_host(ctx, seq, contig_off, n_contigs, genome_of_contig, n_genomes, sp, nullptr, &on_part, subbatch);
    { std::lock_guard<std::mutex> lk(mu); q.push_back(Wave{nullptr, 0, true}); }
    cv.notify_one();
    worker.join();
    if (rc != SK_OK || worker_rc != SK_OK || !keep) { if (merged) sk_sketch_set_free(merged); merged = nullptr; }
    if (rc != SK_OK) return rc;
    if (worker_rc != SK_OK) { ctx->err = "worker: " + worker_err; return worker_rc; }
    if (keep) {
      if (!merged) {   // no genome carried sequence: an empty set of n_genomes sketches
        uint64_t z = 0;
        SK_TRY(sk_sketch_batch(ctx, (const uint8_t*)"", &z, 0, nullptr, n_genomes, sp, &merged));
      }
      *keep = merged;
    }
  }
  SK_CUDA(cudaEventRecord(ev[1], ctx->stream));
  SK_CUDA(cudaEventSynchronize(ev[1]));
  sk_ani_result* o = (sk_ani_result*)malloc(sizeof(sk_ani_result) * (kept.empty() ? 1 : kept.size()));
  if (!o) return SK_ERR_NOMEM;
  if (!kept.empty()) memcpy(o, kept.data(), kept.size() * sizeof(sk_ani_result));
  *out = o; *n_out = kept.size();
  if (stats) {
    float t = 0;
    cudaEventElapsedTime(&t, ev[0], ev[1]);
    memset(stats, 0, sizeof(*stats));
    stats->t_total = t * 1e-3;
    stats->n_pairs_screened = n_screened; stats->n_pairs_kept = kept.size();
  }
  return SK_OK;
}
}  // namespace
