// store_ws.hpp -- working-set execution shared by the host sketch store paths (store.cu: sk_triangle_store,
// sk_query_ref_store; derep.cu: sk_dereplicate_store) and the multi-context calls of multi.cu: the context checks, one host
// thread per context, peer access, the per-context device budget, the markers-only gather of a whole store, chaining global pairs on a
// gathered working set, and chain_working_sets, the one driver that gathers and chains a plan (ws_plan.hpp) on the contexts.
#pragma once
#include <algorithm>
#include <atomic>
#include <chrono>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <string>
#include <thread>
#include <vector>

#include "sk_internal.h"
#include "ws_plan.hpp"

namespace sk {

inline double now_s() { return std::chrono::duration<double>(std::chrono::steady_clock::now().time_since_epoch()).count(); }

// v as a malloc'd array (sk_free; never NULL, also when v is empty)
template <class T>
int hand_out(sk_ctx* ctx, const std::vector<T>& v, T** out, uint64_t* n_out) {
  T* o = (T*)malloc(sizeof(T) * std::max<size_t>(v.size(), 1));
  if (!o) { ctx->err = "out of host memory"; return SK_ERR_NOMEM; }
  if (!v.empty()) memcpy(o, v.data(), v.size() * sizeof(T));
  *out = o; *n_out = v.size();
  return SK_OK;
}

// NULL or repeated contexts (each context gets its own host thread) give SK_ERR_PARAM with the message on ctxs[0]
inline int check_contexts(sk_ctx* const* ctxs, uint32_t n_ctx) {
  for (uint32_t d = 0; d < n_ctx; d++) {
    if (!ctxs[d]) { ctxs[0]->err = "context " + std::to_string(d) + ": NULL context"; return SK_ERR_PARAM; }
    for (uint32_t e = 0; e < d; e++)
      if (ctxs[e] == ctxs[d]) { ctxs[0]->err = "context " + std::to_string(d) + ": the same context appears twice (one host thread per context)"; return SK_ERR_PARAM; }
  }
  return SK_OK;
}

// peer access between the distinct devices of ctxs[0..n) (ignored when unsupported: copies then stage through the host)
inline void enable_peer_access(sk_ctx* const* ctxs, uint32_t n) {
  for (uint32_t a = 0; a < n; a++)
    for (uint32_t b = 0; b < n; b++)
      if (ctxs[a]->device != ctxs[b]->device) {
        cudaSetDevice(ctxs[a]->device);
        int can = 0;
        if (cudaDeviceCanAccessPeer(&can, ctxs[a]->device, ctxs[b]->device) == cudaSuccess && can) cudaDeviceEnablePeerAccess(ctxs[b]->device, 0);
        cudaGetLastError();
      }
}

// fn(d) on one host thread per context (inline for one context), ctxs[d]'s device current.  The call fails if any context
// failed, with the first failing context's code and its message on ctxs[0] as "context d: ...".  ctxs[0]'s device is current
// afterwards.
template <class F>
int run_per_context(sk_ctx* const* ctxs, uint32_t n_ctx, F fn) {
  std::vector<int> rcs(n_ctx, SK_OK);
  auto one = [&](uint32_t d) {
    if (cudaSetDevice(ctxs[d]->device) != cudaSuccess) { ctxs[d]->err = "cudaSetDevice failed"; rcs[d] = SK_ERR_CUDA; }
    else rcs[d] = fn(d);
  };
  if (n_ctx == 1) one(0);
  else {
    std::vector<std::thread> th;
    for (uint32_t d = 0; d < n_ctx; d++) th.emplace_back(one, d);
    for (auto& t : th) t.join();
  }
  cudaSetDevice(ctxs[0]->device);
  for (uint32_t d = 0; d < n_ctx; d++)
    if (rcs[d] != SK_OK) { if (d) ctxs[0]->err = "context " + std::to_string(d) + ": " + ctxs[d]->err; return rcs[d]; }
  return SK_OK;
}

// One host thread per context takes the working sets [0, n_sets) in plan order through an atomic counter: work(d, w) runs
// working set w on ctxs[d].  The first failure stops every context.
template <class F>
int run_working_sets(sk_ctx* const* ctxs, uint32_t n_ctx, size_t n_sets, F work) {
  std::atomic<size_t> next{0};
  std::atomic<bool> failed{false};
  return run_per_context(ctxs, n_ctx, [&](uint32_t d) -> int {
    for (size_t w; !failed && (w = next.fetch_add(1)) < n_sets;) {
      const int rc = work(d, w);
      if (rc != SK_OK) { failed = true; return rc; }
    }
    return SK_OK;
  });
}

// budget per context: a working set's sketches, its gather blob (as large) and the chaining workspace share the device with
// the other contexts on it, so a third of each context's share of the free memory (80 % of it)
inline int working_set_budget(sk_ctx* const* ctxs, uint32_t n_ctx, uint64_t device_budget, uint64_t* budget) {
  *budget = device_budget;
  if (device_budget) return SK_OK;
  sk_ctx* ctx = ctxs[0];
  uint64_t b = ~0ull;
  for (uint32_t d = 0; d < n_ctx; d++) {
    uint32_t same = 0;
    for (uint32_t e = 0; e < n_ctx; e++) same += ctxs[e]->device == ctxs[d]->device;
    size_t free_b = 0, total_b = 0;
    SK_CUDA(cudaSetDevice(ctxs[d]->device));
    SK_CUDA(cudaMemGetInfo(&free_b, &total_b));
    b = std::min<uint64_t>(b, (uint64_t)(0.8 * (double)free_b / (3.0 * same)));
  }
  SK_CUDA(cudaSetDevice(ctx->device));
  *budget = b;
  return SK_OK;
}

// every genome of a store, markers only (the marker screen's input), on ctx
inline int gather_markers(sk_ctx* ctx, const sk_sketch_store* st, sk_sketch_set** out) {
  std::vector<uint32_t> all(sk_sketch_store_n_genomes(st));
  for (uint32_t g = 0; g < all.size(); g++) all[g] = g;
  return sk_sketch_store_gather(ctx, st, all.data(), (uint32_t)all.size(), SK_PACK_MARKERS_ONLY, out);
}

// Chains global pairs (i << 32 | j) on a working set: A holds the genomes a_ids and B the genomes b_ids (both ascending), so
// i and j become indices into them, and the rows' ref_id / query_id are mapped back to global ids.  rows[k] is
// global_pairs[k]'s result whatever its ani.
inline int chain_on_working_set(sk_ctx* c, const sk_sketch_set* A, const std::vector<uint32_t>& a_ids, const sk_sketch_set* B,
                                const std::vector<uint32_t>& b_ids, const std::vector<uint64_t>& global_pairs, const sk_map_params* mp,
                                std::vector<sk_ani_result>& rows) {
  std::vector<uint64_t> lp(global_pairs.size());
  for (size_t i = 0; i < lp.size(); i++) {
    const uint64_t x = std::lower_bound(a_ids.begin(), a_ids.end(), (uint32_t)(global_pairs[i] >> 32)) - a_ids.begin();
    const uint64_t y = std::lower_bound(b_ids.begin(), b_ids.end(), (uint32_t)global_pairs[i]) - b_ids.begin();
    lp[i] = (x << 32) | y;
  }
  rows.resize(lp.size());
  SK_TRY(sk_chain_pairs(c, A, B, lp.data(), lp.size(), mp, rows.data()));
  for (auto& r : rows) { r.ref_id = a_ids[r.ref_id]; r.query_id = b_ids[r.query_id]; }
  return SK_OK;
}

// the genome lists a working set gathers as its reference and query sides: a triangle working set's one list is both
inline const std::vector<uint32_t>& ref_ids(const skws::WorkingSet& ws) { return ws.genomes; }
inline const std::vector<uint32_t>& query_ids(const skws::WorkingSet& ws) { return ws.genomes; }
inline const std::vector<uint32_t>& ref_ids(const skws::QrWorkingSet& ws) { return ws.refs; }
inline const std::vector<uint32_t>& query_ids(const skws::QrWorkingSet& ws) { return ws.queries; }

// The working sets of plan (a skws::Plan or skws::QrPlan) gathered and chained by the contexts in plan order
// (run_working_sets).  A working set's references are gathered from store a and its queries from store b; a triangle working
// set is gathered once, as one set that is both sides.  sink(d, ws, rows) gets rows[k] = ws.pairs[k]'s result with global ids
// on context d's thread.  The plan's counts, the gathered bytes and the gather and chain times are added into stats;
// SK_TRACE=1 prints one line per working set, "[who] context d: working set w/n: ...".
template <class Plan, class Sink>
int chain_working_sets(const char* who, sk_ctx* const* ctxs, uint32_t n_ctx, const sk_sketch_store* a, const sk_sketch_store* b,
                       const Plan& plan, const sk_map_params* mp, Sink sink, sk_store_stats& stats) {
  const bool trace = getenv("SK_TRACE") != nullptr;
  struct Times { double gather = 0, chain = 0; uint64_t bytes = 0; };
  std::vector<Times> times(n_ctx);
  SK_TRY(run_working_sets(ctxs, n_ctx, plan.sets.size(), [&](uint32_t d, size_t w) -> int {
    sk_ctx* c = ctxs[d];
    const auto& ws = plan.sets[w];
    const std::vector<uint32_t>& R = ref_ids(ws);
    const std::vector<uint32_t>& Q = query_ids(ws);
    const bool one = &R == &Q;
    const double t0 = now_s();
    sk_sketch_set *A = nullptr, *B = nullptr;
    int rc = sk_sketch_store_gather(c, a, R.data(), (uint32_t)R.size(), 0, &A);
    if (rc == SK_OK && !one) rc = sk_sketch_store_gather(c, b, Q.data(), (uint32_t)Q.size(), 0, &B);
    const double t1 = now_s();
    if (rc == SK_OK) {
      std::vector<sk_ani_result> rows;
      rc = chain_on_working_set(c, A, R, one ? A : B, Q, ws.pairs, mp, rows);
      if (rc == SK_OK) sink(d, ws, rows);
    }
    if (A) sk_sketch_set_free(A);
    if (B) sk_sketch_set_free(B);
    const double t2 = now_s();
    times[d].gather += t1 - t0; times[d].chain += t2 - t1; times[d].bytes += ws.bytes;
    if (trace) {
      char sides[64];
      if (one) snprintf(sides, sizeof(sides), "%zu genomes", R.size());
      else snprintf(sides, sizeof(sides), "%zu references, %zu queries", R.size(), Q.size());
      fprintf(stderr, "[%s] context %u: working set %zu/%zu%s: %s, %zu pairs, %.1f MB gathered in %.1f ms, chain %.1f ms\n", who, d, w + 1,
              plan.sets.size(), ws.chunk_pair ? " (chunk pair)" : "", sides, ws.pairs.size(), ws.bytes / 1e6, (t1 - t0) * 1e3, (t2 - t1) * 1e3);
    }
    return rc;
  }));
  stats.n_working_sets += (uint32_t)plan.sets.size();
  stats.n_split_components += plan.n_split_components;
  for (const auto& ws : plan.sets) stats.max_working_set_bytes = std::max(stats.max_working_set_bytes, ws.bytes);
  for (const Times& t : times) { stats.gathered_bytes += t.bytes; stats.t_gather += t.gather; stats.t_chain += t.chain; }
  return SK_OK;
}

}  // namespace sk
