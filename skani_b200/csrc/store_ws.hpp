// store_ws.hpp -- working-set execution shared by the host sketch store paths (store.cu: sk_triangle_store,
// sk_query_ref_store; derep.cu: sk_dereplicate_store): the context checks, the per-context device budget and one host
// thread per context taking the planned working sets in order.
#pragma once
#include <algorithm>
#include <atomic>
#include <string>
#include <thread>
#include <vector>

#include "sk_internal.h"

namespace sk {

// NULL or repeated contexts (each context gets its own host thread) give SK_ERR_PARAM with the message on ctxs[0]
inline int check_contexts(sk_ctx* const* ctxs, uint32_t n_ctx) {
  for (uint32_t d = 0; d < n_ctx; d++) {
    if (!ctxs[d]) { ctxs[0]->err = "context " + std::to_string(d) + ": NULL context"; return SK_ERR_PARAM; }
    for (uint32_t e = 0; e < d; e++)
      if (ctxs[e] == ctxs[d]) { ctxs[0]->err = "context " + std::to_string(d) + ": the same context appears twice (one host thread per context)"; return SK_ERR_PARAM; }
  }
  return SK_OK;
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

struct WsTimes { double gather = 0, chain = 0; uint64_t bytes = 0; };

// One host thread per context takes the working sets [0, n_sets) in plan order through an atomic counter;
// work(c, d, w, kept, times) gathers and chains working set w on context c = ctxs[d] and appends the results it keeps.  The
// first failure stops every context and its message goes to ctxs[0].  res: every kept result, sorted by (ref_id, query_id).
template <class F>
int run_working_sets(sk_ctx* const* ctxs, uint32_t n_ctx, size_t n_sets, F work, std::vector<sk_ani_result>& res, WsTimes& total) {
  sk_ctx* ctx = ctxs[0];
  std::atomic<size_t> next{0};
  std::atomic<bool> failed{false};
  std::vector<std::vector<sk_ani_result>> kept(n_ctx);
  std::vector<WsTimes> times(n_ctx);
  std::vector<int> rcs(n_ctx, SK_OK);
  auto run = [&](uint32_t d) {
    sk_ctx* c = ctxs[d];
    if (cudaSetDevice(c->device) != cudaSuccess) { c->err = "cudaSetDevice failed"; rcs[d] = SK_ERR_CUDA; failed = true; return; }
    for (size_t w; !failed && (w = next.fetch_add(1)) < n_sets;) {
      const int rc = work(c, d, w, kept[d], times[d]);
      if (rc != SK_OK) { rcs[d] = rc; failed = true; }
    }
  };
  if (n_ctx == 1) run(0);
  else {
    std::vector<std::thread> th;
    for (uint32_t d = 0; d < n_ctx; d++) th.emplace_back(run, d);
    for (auto& t : th) t.join();
  }
  cudaSetDevice(ctx->device);
  for (uint32_t d = 0; d < n_ctx; d++)
    if (rcs[d] != SK_OK) { if (d) ctx->err = "context " + std::to_string(d) + ": " + ctxs[d]->err; return rcs[d]; }
  for (uint32_t d = 0; d < n_ctx; d++) {
    res.insert(res.end(), kept[d].begin(), kept[d].end());
    total.gather += times[d].gather; total.chain += times[d].chain; total.bytes += times[d].bytes;
  }
  std::sort(res.begin(), res.end(), [](const sk_ani_result& a, const sk_ani_result& b) { return a.ref_id != b.ref_id ? a.ref_id < b.ref_id : a.query_id < b.query_id; });
  return SK_OK;
}

}  // namespace sk
