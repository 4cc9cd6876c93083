// derep.cu -- sk_dereplicate: sk_cluster's greedy representatives of an in-memory sketch set without the triangle.
//
// Genomes are visited in rank order in waves.  A uint8 state per genome (CL_UNDECIDED / CL_REP / CL_MEMBER) stays on the
// device for the whole call.  Per wave:
//   1. the wave's genomes are screened against the representative index (the markers of the representatives chosen so far)
//      and the passing pairs chained; dr_mark_kernel makes every wave genome with an edge to one of them a member.  Every
//      earlier representative ranks before the wave, so such an edge decides the genome; the others may still meet a
//      representative chosen earlier in this wave.
//   2. U = the wave's genomes still undecided.  A temporary index of U's markers screens the pairs inside U (each unordered
//      pair once), they are chained, and sk_cluster's greedy rounds run over U as the frontier on a CSR of those edges.  A
//      genome of U has no edge to an earlier representative, and its edges to members do not matter, so the CSR of U's own
//      edges decides it exactly as the full triangle's graph would.
//   3. the new representatives' markers are sorted and merged into the index (cub::DeviceMerge).
// Then every member is screened against the complete index; the pairs not chained during the waves (a set difference on the
// sorted pair keys) are chained, and cl_assign over the graph of every chained row gives each member its representative.  The
// chained rows contain every edge that touches a representative, which is all the greedy rule reads, so the outcome is
// sk_cluster's on the triangle's rows.
//
// The index is one sorted array of dr_key(marker, slot) (derep_core.cuh) with 16-bit prefix buckets, as the pipelined
// triangle's TriScreen keeps it.  dr_rows_kernel runs one block per row genome and counts shared markers per slot in
// shared-memory tiles; every slot of a tile is then decided by the oriented predicate (dr_screen_pass), so a slot with no
// shared marker that the rescue lets through is emitted like any other.
//
// sk_dereplicate_store runs the same waves over a host sketch store: the markers of every genome are gathered once on ctxs[0]
// (the index, the row screens, the greedy rounds and the set difference run there exactly as above, on the global genome
// indices), and each chain step's pairs are planned into working sets (ws_plan.hpp) that the contexts gather from the store
// and chain through chain_working_sets (store_ws.hpp), as sk_triangle_store does.
//
// sk_dereplicate_fixed and sk_dereplicate_store_fixed start from fixed representatives, the genomes of rank < n_fixed: their
// states are CL_REP and their markers fill the index before the first wave, and the waves cover ranks n_fixed .. N - 1 only.
// No fixed genome is a row of any screen (step 1 and the final screen read wave genomes and members, step 2 undecided wave
// genomes), so no pair of two fixed genomes is screened or chained, and the outcome is sk_cluster's on the triangle's rows
// without those pairs.  sk_dereplicate is n_fixed = 0: the same calls, the same launches.
#include <cub/cub.cuh>

#include <algorithm>
#include <chrono>
#include <cmath>
#include <string>
#include <vector>

#include "cluster_core.cuh"
#include "derep_core.cuh"
#include "sk_internal.h"
#include "store_ws.hpp"
#include "ws_plan.hpp"

using namespace sk;

namespace {

const char* const WHO = "sk_dereplicate";
constexpr int TPB = 256;
// default wave sizes: the first wave holds 64 genomes and each next one twice as many, up to 4096.  Early waves meet few
// representatives, so most of their genomes reach step 2, where every family met twice in one wave chains its pairs
// among itself; later waves are mostly members decided in step 1, and larger waves need fewer host round trips.
constexpr uint32_t FIRST_WAVE = 64, MAX_WAVE = 4096;
constexpr uint32_t TILE = 48 * 1024;   // slots counted per shared-memory tile (192 KiB)

inline unsigned blocks_for(uint64_t n) { return (unsigned)std::max<uint64_t>(1, (n + TPB - 1) / TPB); }
using clk = std::chrono::steady_clock;
inline double secs(clk::time_point t0) { return std::chrono::duration<double>(clk::now() - t0).count(); }

// the keys of list[s]'s markers, slot slot0 + s, at kofs[s] (the exclusive prefix of the list's marker counts)
__global__ void dr_keys_kernel(const uint64_t* __restrict__ markers, const uint64_t* __restrict__ off, const uint32_t* __restrict__ list,
                               const uint64_t* __restrict__ kofs, uint32_t slot0, uint64_t* __restrict__ keys) {
  const uint32_t s = blockIdx.x, g = list[s];
  const uint64_t b = off[g], e = off[g + 1], at = kofs[s];
  for (uint64_t i = b + threadIdx.x; i < e; i += blockDim.x) keys[at + i - b] = dr_key(markers[i], slot0 + s);
}

// bucket[p] = first index position whose key prefix is >= p; bucket[2^16] = n
__global__ void dr_bucket_kernel(const uint64_t* __restrict__ key, uint64_t n, uint32_t* __restrict__ bucket) {
  const uint32_t p = blockIdx.x * blockDim.x + threadIdx.x;
  if (p > (1u << DR_PREFIX_BITS)) return;
  uint64_t lo = 0, hi = n;
  while (lo < hi) {
    const uint64_t mid = (lo + hi) >> 1;
    if ((key[mid] >> DR_PREFIX_SHIFT) < p) lo = mid + 1; else hi = mid;
  }
  bucket[p] = (uint32_t)lo;
}

// One block per row genome rows[k]; columns are the index's slots (upper: only slots > k, for an index whose slot k is row k).
// For each marker of the row the run of that marker is walked from slot t0 to t1 (keys are sorted by marker, then slot).
__global__ void __launch_bounds__(256)
dr_rows_kernel(const uint64_t* __restrict__ markers, const uint64_t* __restrict__ off, const uint32_t* __restrict__ rows,
               const uint64_t* __restrict__ key, uint64_t n_keys, const uint32_t* __restrict__ bucket,
               const uint32_t* __restrict__ slot_genome, uint32_t n_slots, int upper, int rescue_small, double cutoff,
               uint32_t tile, uint64_t* __restrict__ pairs, unsigned long long* __restrict__ n_pairs, unsigned long long cap) {
  extern __shared__ uint32_t counts[];
  const uint32_t k = blockIdx.x, g = rows[k];
  const uint64_t mb = off[g], me = off[g + 1], card_g = me - mb;
  for (uint32_t t0 = upper ? k + 1 : 0; t0 < n_slots; t0 += tile) {
    const uint32_t t1 = min(n_slots, t0 + tile);
    for (uint32_t c = threadIdx.x; c < t1 - t0; c += blockDim.x) counts[c] = 0;
    __syncthreads();
    for (uint64_t e = mb + threadIdx.x; e < me; e += blockDim.x) {
      const uint64_t m = markers[e], k0 = dr_key(m, t0), k1 = dr_key(m, t1);
      const uint32_t p = (uint32_t)(k0 >> DR_PREFIX_SHIFT);
      uint64_t lo = bucket[p], hi = bucket[p + 1];
      while (lo < hi) {
        const uint64_t mid = (lo + hi) >> 1;
        if (key[mid] < k0) lo = mid + 1; else hi = mid;
      }
      for (uint64_t t = lo; t < n_keys; t++) {
        const uint64_t kk = key[t];
        if (kk >= k1) break;
        atomicAdd(&counts[dr_key_slot(kk) - t0], 1u);
      }
    }
    __syncthreads();
    for (uint32_t c = threadIdx.x; c < t1 - t0; c += blockDim.x) {
      const uint32_t r = slot_genome[t0 + c];
      if (dr_screen_pass(g, card_g, r, off[r + 1] - off[r], counts[c], rescue_small, cutoff)) {
        const unsigned long long at = atomicAdd(n_pairs, 1ull);
        if (at < cap) pairs[at] = dr_pair_key(g, r);
      }
    }
    __syncthreads();
  }
}

// step 1: the wave genome of every chained row that is an edge becomes a member (the row's other genome is a representative)
__global__ void dr_mark_kernel(const sk_ani_result* __restrict__ rows, uint64_t m, float min_ani, uint8_t* state) {
  const uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= m) return;
  const sk_ani_result& r = rows[i];
  if (!cl_is_edge(r.ani, min_ani)) return;
  state[state[r.ref_id] == CL_REP ? r.query_id : r.ref_id] = CL_MEMBER;
}

struct HasState {
  const uint8_t* state;
  uint8_t s;
  __device__ bool operator()(uint32_t v) const { return state[v] == s; }
};

// the set difference of the final screen: a pair is kept unless the sorted chained keys hold it
struct NotChained {
  const uint64_t* chained;
  uint64_t n;
  __device__ bool operator()(uint64_t k) const {
    uint64_t lo = 0, hi = n;
    while (lo < hi) {
      const uint64_t mid = (lo + hi) >> 1;
      if (chained[mid] < k) lo = mid + 1; else hi = mid;
    }
    return lo == n || chained[lo] != k;
  }
};

// a marker index over slots 0 .. slots - 1 (slot s = genome slot_genome[s]).  Its slots may all be without markers: the
// buckets then stay zero and n = 0, so no row walks the (absent) keys.
struct Index {
  DTmp<uint64_t> key[2];
  int cur = 0;
  uint64_t n = 0;
  DTmp<uint32_t> bucket, slot_genome;
  uint32_t slots = 0;
};

// a cub call run twice: sizing, then on temporaries from the arena
template <typename F>
int cub_run(sk_ctx* ctx, const char* who, const char* what, F&& f) {
  size_t tb = 0;
  SK_CUDA(f((void*)nullptr, tb));
  DTmp<uint8_t> tmp;
  SK_TRY(cl_alloc(ctx, tmp, tb, what, who));
  SK_CUDA(f((void*)tmp.p, tb));
  count_launch(ctx, 1);
  return SK_OK;
}

// chain()'s host sketch store back end (sk_dereplicate_store): the sketches of every genome in a store, the contexts that
// chain, the working-set budget per context and the sk_store_stats summed over the chain steps
struct StoreChain {
  sk_ctx* const* ctxs;
  uint32_t n_ctx;
  const sk_sketch_store* st;
  std::vector<uint64_t> gbytes;   // sk_sketch_store_genome_bytes of every genome
  uint64_t budget;
  sk_store_stats stats{};
};

// set: the markers (and mk_off) of every genome, which the index, the row screens and the key offsets read; it is also what
// chain() chains unless `store` is set, in which case set may hold the markers only (a SK_PACK_MARKERS_ONLY gather)
struct Run {
  sk_ctx* ctx;
  const sk_sketch_set* set;
  const sk_map_params* mp;
  float min_ani;
  double cutoff;
  uint32_t N;
  const char* who = WHO;
  StoreChain* store = nullptr;
  DTmp<uint64_t> d_off;
  DTmp<uint32_t> d_rank;
  DTmp<uint8_t> state;
  std::vector<sk_ani_result> rows;   // every chained row, in chaining order
  std::vector<uint64_t> chained;     // their pair keys
  sk_derep_stats st{};

  // every genome's marker offsets on the device (d_off), which the index and the row screens read
  int upload_offsets() {
    SK_TRY(cl_alloc(ctx, d_off, (uint64_t)N + 1, "marker offsets", who));
    SK_CUDA(h2d_small(ctx, d_off.p, set->mk_off.data(), ((size_t)N + 1) * 8));
    return SK_OK;
  }

  // genomes list[0 .. m) (host; d_list the same on the device) join ix as slots ix.slots ..
  int index_add(Index& ix, const uint32_t* list, const uint32_t* d_list, uint32_t m) {
    if (!m) return SK_OK;
    cudaStream_t s = ctx->stream;
    std::vector<uint64_t> kofs(m + 1, 0);
    for (uint32_t i = 0; i < m; i++) kofs[i + 1] = kofs[i] + set->mk_off[list[i] + 1] - set->mk_off[list[i]];
    const uint64_t m_new = kofs[m], n_tot = ix.n + m_new;
    if ((uint64_t)ix.slots + m > DR_MAX_SLOTS) {
      ctx->err = std::string(who) + ": more than 2^22 - 1 genomes (" + std::to_string((uint64_t)ix.slots + m) + ") in one marker index"; return SK_ERR_PARAM;
    }
    if (n_tot >= DR_MAX_KEYS) {
      ctx->err = std::string(who) + ": " + std::to_string(n_tot) + " markers in one marker index (at most 2^31 - 1)"; return SK_ERR_PARAM;
    }
    SK_CUDA(cudaMemcpyAsync(ix.slot_genome.p + ix.slots, d_list, (size_t)m * 4, cudaMemcpyDeviceToDevice, s));
    if (m_new) {
      DTmp<uint64_t> d_kofs, nk, snk;
      SK_TRY(cl_alloc(ctx, d_kofs, m + 1, "key offsets", who));
      SK_TRY(cl_alloc(ctx, nk, m_new, "index keys", who));
      SK_TRY(cl_alloc(ctx, snk, m_new, "index keys", who));
      SK_CUDA(h2d_small(ctx, d_kofs.p, kofs.data(), (size_t)(m + 1) * 8));
      dr_keys_kernel<<<m, 256, 0, s>>>(set->markers, d_off.p, d_list, d_kofs.p, ix.slots, nk.p);
      count_launch(ctx, 1);
      SK_CUDA(cudaGetLastError());
      SK_TRY(cub_run(ctx, who, "index sort", [&](void* t, size_t& tb) {
        return cub::DeviceRadixSort::SortKeys(t, tb, nk.p, snk.p, (int)m_new, 0, 64, s); }));
      DTmp<uint64_t>& dst = ix.key[ix.cur ^ 1];
      SK_TRY(cl_alloc(ctx, dst, n_tot, "marker index", who));
      if (!ix.n) {
        SK_CUDA(cudaMemcpyAsync(dst.p, snk.p, m_new * 8, cudaMemcpyDeviceToDevice, s));
      } else {   // keys are distinct (marker, slot) pairs: the merge has one possible output
        const uint64_t* old = ix.key[ix.cur].p;
        SK_TRY(cub_run(ctx, who, "index merge", [&](void* t, size_t& tb) {
          return cub::DeviceMerge::MergeKeys(t, tb, old, (int)ix.n, snk.p, (int)m_new, dst.p, ::cuda::std::less<uint64_t>{}, s); }));
      }
      ix.cur ^= 1;
      ix.key[ix.cur ^ 1].release();
      ix.n = n_tot;
      dr_bucket_kernel<<<((1u << DR_PREFIX_BITS) + 256) / 256, 256, 0, s>>>(ix.key[ix.cur].p, ix.n, ix.bucket.p);
      count_launch(ctx, 1);
      SK_CUDA(cudaGetLastError());
      SK_CUDA(cudaStreamSynchronize(s));   // the temporaries go back to the arena
    }
    ix.slots += m;
    return SK_OK;
  }

  // the pairs (d_rows[k], slot genome) that pass the triangle's screen, sorted, on the device in out[0 .. *n_out)
  int screen(const Index& ix, const uint32_t* d_rows, uint32_t n_rows, bool upper, DTmp<uint64_t>& out, uint64_t* n_out) {
    const auto t0 = clk::now();
    cudaStream_t s = ctx->stream;
    *n_out = 0;
    if (!n_rows || !ix.slots) { st.t_screen += secs(t0); return SK_OK; }
    const uint32_t tile = std::min(ix.slots, TILE);
    SK_CUDA(cudaFuncSetAttribute(dr_rows_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, TILE * 4));   // constant: see run_screen
    unsigned long long cap = std::max<unsigned long long>(1ull << 20, 64ull * n_rows), n = 0;
    DTmp<unsigned long long> d_n;
    DTmp<uint64_t> d_pairs;
    SK_TRY(cl_alloc(ctx, d_n, 1, "pair count", who));
    for (int attempt = 0; attempt < 2; attempt++) {
      SK_TRY(cl_alloc(ctx, d_pairs, cap, "screened pairs", who));
      SK_CUDA(cudaMemsetAsync(d_n.p, 0, 8, s));
      SK_LAUNCH(ctx, "dr_rows_kernel", (dr_rows_kernel<<<n_rows, 256, (size_t)tile * 4, s>>>(
          set->markers, d_off.p, d_rows, ix.key[ix.cur].p, ix.n, ix.bucket.p, ix.slot_genome.p, ix.slots, upper, mp->rescue_small, cutoff,
          tile, d_pairs.p, d_n.p, cap)));
      SK_CUDA(cudaGetLastError());
      SK_CUDA(cudaMemcpyAsync(&n, d_n.p, 8, cudaMemcpyDeviceToHost, s));
      SK_CUDA(cudaStreamSynchronize(s));
      if (n <= cap) break;
      cap = n;
    }
    SK_TRY(cl_alloc(ctx, out, n, "screened pairs", who));
    if (n) SK_TRY(cub_run(ctx, who, "pair sort", [&](void* t, size_t& tb) {
      return cub::DeviceRadixSort::SortKeys(t, tb, d_pairs.p, out.p, (int)n, 0, 64, s); }));
    SK_CUDA(cudaStreamSynchronize(s));
    *n_out = n;
    st.pairs_screened += n;
    st.t_screen += secs(t0);
    return SK_OK;
  }

  // d_pairs[0 .. n) (device, sorted) chained as the triangle chains them; the rows are appended to `rows`, the first at *first,
  // row i of the step being pair i's whatever its ani
  int chain(const uint64_t* d_pairs, uint64_t n, size_t* first) {
    *first = rows.size();
    if (!n) return SK_OK;
    const auto t0 = clk::now();
    std::vector<uint64_t> pairs(n);
    SK_CUDA(cudaMemcpyAsync(pairs.data(), d_pairs, n * 8, cudaMemcpyDeviceToHost, ctx->stream));
    SK_CUDA(cudaStreamSynchronize(ctx->stream));
    rows.resize(*first + n);
    if (store) SK_TRY(chain_store(pairs, rows.data() + *first));
    else SK_TRY(sk_chain_pairs(ctx, set, set, pairs.data(), n, mp, rows.data() + *first));
    chained.insert(chained.end(), pairs.begin(), pairs.end());
    st.pairs_chained += n;
    st.t_chain += secs(t0);
    return SK_OK;
  }

  // The store back end: the step's sorted pairs planned into working sets (ws_plan.hpp) that the contexts gather and chain
  // (chain_working_sets), as sk_triangle_store does.  Each pair is in exactly one working set and its row goes to the pair's
  // position in out, so the contexts never write the same row and out does not depend on which context chained what.
  int chain_store(const std::vector<uint64_t>& pairs, sk_ani_result* out) {
    StoreChain& sc = *store;
    skws::Plan plan;
    std::string perr;
    if (!skws::plan_working_sets(pairs, sc.gbytes, sc.budget, plan, perr)) { ctx->err = std::string(who) + ": " + perr; return SK_ERR_NOMEM; }
    return chain_working_sets(who, sc.ctxs, sc.n_ctx, sc.st, sc.st, plan, mp, [&](uint32_t, const skws::WorkingSet& ws, const std::vector<sk_ani_result>& res) {
      for (size_t i = 0; i < res.size(); i++) out[std::lower_bound(pairs.begin(), pairs.end(), ws.pairs[i]) - pairs.begin()] = res[i];
    }, sc.stats);
  }

  // the genomes of list[0 .. m) (device) in state s, order kept, into out; their count
  int select(const uint32_t* list, uint32_t m, uint8_t s, DTmp<uint32_t>& out, uint32_t* n_out) {
    DTmp<uint32_t> d_m;
    SK_TRY(cl_alloc(ctx, out, m, "genome list", who));
    SK_TRY(cl_alloc(ctx, d_m, 1, "genome count", who));
    *n_out = 0;
    if (!m) return SK_OK;
    SK_TRY(cub_run(ctx, who, "genome selection", [&](void* t, size_t& tb) {
      return cub::DeviceSelect::If(t, tb, list, out.p, d_m.p, (int)m, HasState{state.p, s}, ctx->stream); }));
    SK_CUDA(cudaMemcpyAsync(n_out, d_m.p, 4, cudaMemcpyDeviceToHost, ctx->stream));
    SK_CUDA(cudaStreamSynchronize(ctx->stream));
    return SK_OK;
  }

  int to_host(const DTmp<uint32_t>& d, uint32_t m, std::vector<uint32_t>& h) {
    h.resize(m);
    if (m) SK_CUDA(cudaMemcpyAsync(h.data(), d.p, (size_t)m * 4, cudaMemcpyDeviceToHost, ctx->stream));
    SK_CUDA(cudaStreamSynchronize(ctx->stream));
    return SK_OK;
  }

  // wave = genomes per wave, 0 for the growing default; the genomes of rank < n_fixed are representatives from the start
  int run(const uint32_t* rank, uint32_t n_fixed, uint32_t wave, uint32_t* rep, uint32_t* cluster, sk_ani_result* join) {
    cudaStream_t s = ctx->stream;
    const auto t_all = clk::now();
    std::vector<uint32_t> order(N);
    for (uint32_t g = 0; g < N; g++) order[rank[g]] = g;
    uint64_t fixed_markers = 0;
    for (uint32_t i = 0; i < n_fixed; i++) fixed_markers += set->mk_off[order[i] + 1] - set->mk_off[order[i]];
    if (fixed_markers >= DR_MAX_KEYS) {
      ctx->err = std::string(who) + ": the " + std::to_string(n_fixed) + " fixed representatives hold " + std::to_string(fixed_markers) +
                 " markers, more than one marker index takes (at most 2^31 - 1)";
      return SK_ERR_PARAM;
    }
    DTmp<uint32_t> d_order;
    Index reps;
    SK_TRY(upload_offsets());
    SK_TRY(cl_alloc(ctx, d_rank, N, "ranks", who));
    SK_TRY(cl_alloc(ctx, d_order, N, "rank order", who));
    SK_TRY(cl_alloc(ctx, state, N, "states", who));
    SK_TRY(cl_alloc(ctx, reps.bucket, (1u << DR_PREFIX_BITS) + 1, "index buckets", who));
    SK_TRY(cl_alloc(ctx, reps.slot_genome, N, "index slots", who));
    SK_CUDA(cudaMemsetAsync(reps.bucket.p, 0, ((1u << DR_PREFIX_BITS) + 1) * 4, s));
    SK_CUDA(h2d_small(ctx, d_rank.p, rank, (size_t)N * 4));
    SK_CUDA(h2d_small(ctx, d_order.p, order.data(), (size_t)N * 4));
    SK_CUDA(cudaMemsetAsync(state.p, CL_UNDECIDED, N, s));
    // the fixed representatives: their states and their markers in the index before the first wave
    std::vector<uint8_t> fixed_state;
    if (n_fixed) {
      fixed_state.assign(N, CL_UNDECIDED);
      for (uint32_t i = 0; i < n_fixed; i++) fixed_state[order[i]] = CL_REP;
      SK_CUDA(cudaMemcpyAsync(state.p, fixed_state.data(), N, cudaMemcpyHostToDevice, s));
      const auto t0 = clk::now();
      SK_TRY(index_add(reps, order.data(), d_order.p, n_fixed));
      st.t_screen += secs(t0);
    }
    for (uint32_t w0 = n_fixed, size = wave ? wave : FIRST_WAVE; w0 < N; w0 += size, size = wave ? wave : std::min(2 * size, MAX_WAVE)) {
      const uint32_t w1 = std::min<uint64_t>(N, (uint64_t)w0 + size), nw = w1 - w0;
      const uint32_t* d_wave = d_order.p + w0;
      st.waves++;
      // 1. the wave against the representatives chosen so far
      DTmp<uint64_t> pairs;
      uint64_t np = 0;
      size_t first = 0;
      SK_TRY(screen(reps, d_wave, nw, false, pairs, &np));
      SK_TRY(chain(pairs.p, np, &first));
      const auto t_mark = clk::now();
      if (np) {
        DTmp<sk_ani_result> d_res;
        SK_TRY(cl_alloc(ctx, d_res, np, "chained rows", who));
        SK_TRY(upload_runs(ctx, (uint8_t*)d_res.p, {{(const uint8_t*)(rows.data() + first), np * sizeof(sk_ani_result)}}, false));
        dr_mark_kernel<<<blocks_for(np), TPB, 0, s>>>(d_res.p, np, min_ani, state.p);
        count_launch(ctx, 1);
        SK_CUDA(cudaGetLastError());
      }
      DTmp<uint32_t> d_u;
      uint32_t nu = 0;
      SK_TRY(select(d_wave, nw, CL_UNDECIDED, d_u, &nu));
      st.t_decide += secs(t_mark);
      if (!nu) continue;
      // 2. inside the wave: U screened against a temporary index of its own markers, each pair once
      std::vector<uint32_t> u;
      SK_TRY(to_host(d_u, nu, u));
      {
        Index ui;
        SK_TRY(cl_alloc(ctx, ui.bucket, (1u << DR_PREFIX_BITS) + 1, "index buckets", who));
        SK_TRY(cl_alloc(ctx, ui.slot_genome, nu, "index slots", who));
        SK_CUDA(cudaMemsetAsync(ui.bucket.p, 0, ((1u << DR_PREFIX_BITS) + 1) * 4, s));
        const auto t0 = clk::now();
        SK_TRY(index_add(ui, u.data(), d_u.p, nu));
        st.t_screen += secs(t0);
        SK_TRY(screen(ui, d_u.p, nu, true, pairs, &np));
      }
      SK_TRY(chain(pairs.p, np, &first));
      pairs.release();
      const auto t_greedy = clk::now();
      {
        Graph g;
        SK_TRY(build_graph(ctx, who, N, rows.data() + first, np, min_ani, g));
        SK_TRY(greedy_rounds(ctx, who, d_u.p, nu, g, d_rank.p, state.p, &st.rounds));
      }
      // 3. the new representatives join the index
      DTmp<uint32_t> d_new;
      uint32_t nn = 0;
      SK_TRY(select(d_u.p, nu, CL_REP, d_new, &nn));
      st.t_decide += secs(t_greedy);
      std::vector<uint32_t> fresh;
      SK_TRY(to_host(d_new, nn, fresh));
      const auto t0 = clk::now();
      SK_TRY(index_add(reps, fresh.data(), d_new.p, nn));
      st.t_screen += secs(t0);
    }
    // every member against every representative; only the pairs not chained yet are chained
    DTmp<uint32_t> d_mem;
    uint32_t nm = 0;
    SK_TRY(select(d_order.p, N, CL_MEMBER, d_mem, &nm));
    DTmp<uint64_t> pairs, fresh;
    uint64_t np = 0, nf = 0;
    SK_TRY(screen(reps, d_mem.p, nm, false, pairs, &np));
    if (np) {
      const auto t0 = clk::now();
      std::vector<uint64_t> done = chained;
      std::sort(done.begin(), done.end());
      DTmp<uint64_t> d_done;
      DTmp<unsigned long long> d_nf;
      SK_TRY(cl_alloc(ctx, d_done, done.size(), "chained pairs", who));
      SK_TRY(cl_alloc(ctx, fresh, np, "pairs to chain", who));
      SK_TRY(cl_alloc(ctx, d_nf, 1, "pair count", who));
      if (!done.empty()) SK_CUDA(cudaMemcpyAsync(d_done.p, done.data(), done.size() * 8, cudaMemcpyHostToDevice, s));
      SK_TRY(cub_run(ctx, who, "set difference", [&](void* t, size_t& tb) {
        return cub::DeviceSelect::If(t, tb, pairs.p, fresh.p, d_nf.p, (int)np, NotChained{d_done.p, done.size()}, s); }));
      unsigned long long h = 0;
      SK_CUDA(cudaMemcpyAsync(&h, d_nf.p, 8, cudaMemcpyDeviceToHost, s));
      SK_CUDA(cudaStreamSynchronize(s));
      nf = h;
      st.t_screen += secs(t0);
    }
    pairs.release();
    size_t first = 0;
    SK_TRY(chain(fresh.p, nf, &first));
    fresh.release();
    // the assignment over every chained row, representatives numbered in rank order
    const auto t_assign = clk::now();
    Graph g;
    SK_TRY(build_graph(ctx, who, N, rows.data(), rows.size(), min_ani, g));
    DTmp<uint32_t> d_rep, d_cluster, flag;
    DTmp<uint64_t> d_edge;
    SK_TRY(cl_alloc(ctx, d_rep, N, "representatives", who));
    SK_TRY(cl_alloc(ctx, d_cluster, N, "clusters", who));
    SK_TRY(cl_alloc(ctx, flag, N, "flags", who));
    SK_TRY(cl_alloc(ctx, d_edge, N, "edges per genome", who));
    SK_TRY(greedy_assign(ctx, N, g, d_rank.p, state.p, d_rep.p, d_edge.p, flag.p));
    std::vector<uint32_t> h_rep(N), h_cluster(N);   // read back here first: the caller's outputs may alias each other
    std::vector<uint64_t> edge(N);
    SK_TRY(number_and_read_back(ctx, who, N, d_rank.p, d_rep.p, d_edge.p, flag.p, d_cluster.p, h_rep.data(), h_cluster.data(), edge.data(),
                                &st.n_clusters));
    st.t_decide += secs(t_assign);
    st.n_edges = g.E;
    for (uint32_t v = 0; v < N; v++) {
      if (h_rep[v] == v) {
        join[v] = sk_ani_result{};
        join[v].ani = NAN;
        join[v].ref_id = join[v].query_id = v;
      } else if (edge[v] == UINT64_MAX) {
        ctx->err = std::string(who) + ": member " + std::to_string(v) + " has no chained row to its representative";
        return SK_ERR_STATE;
      } else {
        join[v] = rows[edge[v]];
      }
    }
    std::copy(h_rep.begin(), h_rep.end(), rep);
    std::copy(h_cluster.begin(), h_cluster.end(), cluster);
    st.t_total = secs(t_all);
    return SK_OK;
  }
};

// the refusal of a fixed set larger than the representative index, before any device work; empty when it fits
std::string fixed_error(uint32_t n_fixed, uint32_t n_genomes) {
  if (n_fixed > n_genomes)
    return "n_fixed = " + std::to_string(n_fixed) + " fixed representatives, more than the " + std::to_string(n_genomes) + " genomes";
  if (n_fixed > DR_MAX_SLOTS)
    return "n_fixed = " + std::to_string(n_fixed) + " fixed representatives, more than one marker index takes (at most 2^22 - 1)";
  return "";
}

// sk_dereplicate and sk_dereplicate_fixed (who names the caller in messages): sk_dereplicate is n_fixed = 0
int dereplicate_impl(const char* who, sk_ctx* ctx, const sk_sketch_set* set, const sk_map_params* mp, const uint32_t* rank, uint32_t n_fixed,
                     const sk_derep_params* dp, uint32_t* rep, uint32_t* cluster, sk_ani_result* join, sk_derep_stats* stats) {
  if (!ctx) return SK_ERR_PARAM;
  if (!set || !mp || !dp || !rep || !cluster || !join || (set->G && !rank)) { ctx->err = std::string(who) + ": NULL argument"; return SK_ERR_PARAM; }
  if (std::isnan(dp->min_ani)) { ctx->err = std::string(who) + ": min_ani is NaN"; return SK_ERR_PARAM; }
  const std::string bad = rank_error(set->G, rank);
  if (!bad.empty()) { ctx->err = std::string(who) + ": " + bad; return SK_ERR_PARAM; }
  const std::string fbad = fixed_error(n_fixed, set->G);
  if (!fbad.empty()) { ctx->err = std::string(who) + ": " + fbad; return SK_ERR_PARAM; }
  SK_CUDA(cudaSetDevice(ctx->device));
  Run r{ctx, set, mp, dp->min_ani, screen_cutoff(mp), set->G, who};
  const uint32_t wave = std::min(dp->wave, DR_MAX_SLOTS);
  const int rc = r.run(rank, n_fixed, wave, rep, cluster, join);
  if (rc == SK_OK && stats) *stats = r.st;
  return rc;
}

}  // namespace

int sk_dereplicate(sk_ctx* ctx, const sk_sketch_set* set, const sk_map_params* mp, const uint32_t* rank, const sk_derep_params* dp,
                   uint32_t* rep, uint32_t* cluster, sk_ani_result* join, sk_derep_stats* stats) {
  return dereplicate_impl(WHO, ctx, set, mp, rank, 0, dp, rep, cluster, join, stats);
}

int sk_dereplicate_fixed(sk_ctx* ctx, const sk_sketch_set* set, const sk_map_params* mp, const uint32_t* rank, uint32_t n_fixed,
                         const sk_derep_params* dp, uint32_t* rep, uint32_t* cluster, sk_ani_result* join, sk_derep_stats* stats) {
  return dereplicate_impl("sk_dereplicate_fixed", ctx, set, mp, rank, n_fixed, dp, rep, cluster, join, stats);
}

int sk_debug_derep_screen(sk_ctx* ctx, const sk_sketch_set* set, const sk_map_params* mp, const uint32_t* slot_genome,
                          uint32_t n_slots, const uint32_t* batch_sizes, uint32_t n_batches, const uint32_t* rows, uint32_t n_rows,
                          int upper, uint64_t** pairs, uint64_t* n_pairs, uint64_t** keys, uint64_t* n_keys, uint32_t* bucket) {
  const char* const who = "sk_debug_derep_screen";
  if (!ctx) return SK_ERR_PARAM;
  if (!set || !mp || !pairs || !n_pairs || (n_slots && !slot_genome) || (n_batches && !batch_sizes) || (n_rows && !rows) ||
      (!keys != !n_keys)) {
    ctx->err = std::string(who) + ": NULL argument"; return SK_ERR_PARAM;
  }
  const uint32_t G = set->G;
  for (uint32_t i = 0; i < n_slots; i++)
    if (slot_genome[i] >= G) { ctx->err = std::string(who) + ": slot " + std::to_string(i) + " holds genome " + std::to_string(slot_genome[i]) + " >= " + std::to_string(G); return SK_ERR_PARAM; }
  for (uint32_t i = 0; i < n_rows; i++)
    if (rows[i] >= G) { ctx->err = std::string(who) + ": row " + std::to_string(i) + " is genome " + std::to_string(rows[i]) + " >= " + std::to_string(G); return SK_ERR_PARAM; }
  uint64_t sum = 0;
  for (uint32_t b = 0; b < n_batches; b++) sum += batch_sizes[b];
  if (sum != n_slots) { ctx->err = std::string(who) + ": batch sizes sum to " + std::to_string(sum) + ", not n_slots = " + std::to_string(n_slots); return SK_ERR_PARAM; }
  if (upper && (n_rows != n_slots || !std::equal(rows, rows + n_rows, slot_genome))) {
    ctx->err = std::string(who) + ": upper needs rows equal to slot_genome"; return SK_ERR_PARAM;
  }
  SK_CUDA(cudaSetDevice(ctx->device));
  Run r{ctx, set, mp, 0.f, screen_cutoff(mp), G, who};
  SK_TRY(r.upload_offsets());
  Index ix;
  DTmp<uint32_t> d_slots, d_rows;
  SK_TRY(cl_alloc(ctx, ix.bucket, (1u << DR_PREFIX_BITS) + 1, "index buckets", who));
  SK_TRY(cl_alloc(ctx, ix.slot_genome, n_slots, "index slots", who));
  SK_TRY(cl_alloc(ctx, d_slots, n_slots, "slot list", who));
  SK_TRY(cl_alloc(ctx, d_rows, n_rows, "rows", who));
  SK_CUDA(cudaMemsetAsync(ix.bucket.p, 0, ((1u << DR_PREFIX_BITS) + 1) * 4, ctx->stream));
  SK_CUDA(h2d_small(ctx, d_slots.p, slot_genome, (size_t)n_slots * 4));
  SK_CUDA(h2d_small(ctx, d_rows.p, rows, (size_t)n_rows * 4));
  for (uint32_t b = 0, at = 0; b < n_batches; at += batch_sizes[b++]) SK_TRY(r.index_add(ix, slot_genome + at, d_slots.p + at, batch_sizes[b]));
  DTmp<uint64_t> d_pairs;
  uint64_t n = 0;
  SK_TRY(r.screen(ix, d_rows.p, n_rows, upper != 0, d_pairs, &n));
  uint64_t* hp = (uint64_t*)malloc(std::max<uint64_t>(n, 1) * 8);
  uint64_t* hk = keys ? (uint64_t*)malloc(std::max<uint64_t>(ix.n, 1) * 8) : nullptr;
  if (!hp || (keys && !hk)) { free(hp); free(hk); ctx->err = std::string(who) + ": out of host memory"; return SK_ERR_NOMEM; }
  cudaError_t e = cudaSuccess;
  if (n) e = cudaMemcpyAsync(hp, d_pairs.p, n * 8, cudaMemcpyDeviceToHost, ctx->stream);
  if (e == cudaSuccess && hk && ix.n) e = cudaMemcpyAsync(hk, ix.key[ix.cur].p, ix.n * 8, cudaMemcpyDeviceToHost, ctx->stream);
  if (e == cudaSuccess && bucket) e = cudaMemcpyAsync(bucket, ix.bucket.p, ((1u << DR_PREFIX_BITS) + 1) * 4, cudaMemcpyDeviceToHost, ctx->stream);
  if (e == cudaSuccess) e = cudaStreamSynchronize(ctx->stream);
  if (e != cudaSuccess) { free(hp); free(hk); ctx->err = std::string(who) + ": " + cudaGetErrorString(e); return SK_ERR_CUDA; }
  *pairs = hp;
  *n_pairs = n;
  if (keys) { *keys = hk; *n_keys = ix.n; }
  return SK_OK;
}

namespace {

const char* const WHO_STORE = "sk_dereplicate_store";

// sk_dereplicate_store's working-set budget per context when device_budget is 0 (after the marker set is on ctxs[0]):
// working_set_budget's, except that ctxs[0]'s device first keeps room for the representative index at its largest (every
// genome a representative): two key buffers of 8 bytes per marker, the new keys and their sorted copy, the sort's
// temporaries, the per-genome arrays, and 64 MiB for the screens' pair buffers and the buckets
int derep_store_budget(sk_ctx* const* ctxs, uint32_t n_ctx, uint64_t n_markers, uint32_t n_genomes, uint64_t* budget) {
  sk_ctx* ctx = ctxs[0];
  SK_TRY(working_set_budget(ctxs, n_ctx, 0, budget));
  const double reserve = 5.0 * 8.0 * (double)n_markers + 32.0 * n_genomes + (64ull << 20);
  uint32_t same = 0;
  for (uint32_t d = 0; d < n_ctx; d++) same += ctxs[d]->device == ctx->device;
  size_t free_b = 0, total_b = 0;
  SK_CUDA(cudaSetDevice(ctx->device));
  SK_CUDA(cudaMemGetInfo(&free_b, &total_b));
  const double left = std::max(0.0, (double)free_b - reserve);
  *budget = std::min<uint64_t>(*budget, (uint64_t)(0.8 * left / (3.0 * same)));
  return SK_OK;
}

// sk_dereplicate_store and sk_dereplicate_store_fixed (who names the caller in messages): sk_dereplicate_store is n_fixed = 0
int dereplicate_store_impl(const char* who, sk_ctx* const* ctxs, uint32_t n_ctx, const sk_sketch_store* st, const sk_map_params* mp,
                           const uint32_t* rank, uint32_t n_fixed, const sk_derep_params* dp, uint64_t device_budget, uint32_t* rep,
                           uint32_t* cluster, sk_ani_result* join, sk_derep_stats* stats, sk_store_stats* store_stats) {
  if (!ctxs || n_ctx == 0 || !ctxs[0]) return SK_ERR_PARAM;
  sk_ctx* ctx = ctxs[0];
  const uint32_t N = sk_sketch_store_n_genomes(st);
  if (!st || !mp || !dp || !rep || !cluster || !join || (N && !rank)) { ctx->err = std::string(who) + ": NULL argument"; return SK_ERR_PARAM; }
  SK_TRY(check_contexts(ctxs, n_ctx));
  if (std::isnan(dp->min_ani)) { ctx->err = std::string(who) + ": min_ani is NaN"; return SK_ERR_PARAM; }
  const std::string bad = rank_error(N, rank);
  if (!bad.empty()) { ctx->err = std::string(who) + ": " + bad; return SK_ERR_PARAM; }
  const std::string fbad = fixed_error(n_fixed, N);
  if (!fbad.empty()) { ctx->err = std::string(who) + ": " + fbad; return SK_ERR_PARAM; }
  StoreChain sc{ctxs, n_ctx, st, std::vector<uint64_t>(N), device_budget};
  for (uint32_t g = 0; g < N; g++) sc.gbytes[g] = sk_sketch_store_genome_bytes(st, g);
  std::string perr;   // a genome over budget / 2 cannot be placed in every chunk pair of a working-set plan
  if (device_budget && !skws::genomes_fit(sc.gbytes, device_budget, perr)) {   // before any device work
    ctx->err = std::string(who) + ": " + perr;
    return SK_ERR_NOMEM;
  }
  if (N == 0) {   // what sk_dereplicate returns for an empty set: no wave, no pair, no cluster
    if (stats) *stats = sk_derep_stats{};
    if (store_stats) *store_stats = sk_store_stats{};
    return SK_OK;
  }
  // the markers of every genome on ctxs[0]
  SK_CUDA(cudaSetDevice(ctx->device));
  const auto t0 = clk::now();
  sk_sketch_set* mk = nullptr;
  SK_TRY(gather_markers(ctx, st, &mk));
  sc.stats.t_screen = secs(t0);
  int rc = SK_OK;
  if (!device_budget) {
    rc = derep_store_budget(ctxs, n_ctx, mk->mk_off[N], N, &sc.budget);
    if (rc == SK_OK && !skws::genomes_fit(sc.gbytes, sc.budget, perr)) { ctx->err = std::string(who) + ": " + perr; rc = SK_ERR_NOMEM; }
  }
  if (rc == SK_OK) {
    Run r{ctx, mk, mp, dp->min_ani, screen_cutoff(mp), N, who, &sc};
    rc = r.run(rank, n_fixed, std::min(dp->wave, DR_MAX_SLOTS), rep, cluster, join);
    r.st.t_total += sc.stats.t_screen;
    if (rc == SK_OK && stats) *stats = r.st;
  }
  sk_sketch_set_free(mk);
  if (rc == SK_OK && store_stats) *store_stats = sc.stats;
  return rc;
}

}  // namespace

int sk_dereplicate_store(sk_ctx* const* ctxs, uint32_t n_ctx, const sk_sketch_store* st, const sk_map_params* mp, const uint32_t* rank,
                         const sk_derep_params* dp, uint64_t device_budget, uint32_t* rep, uint32_t* cluster, sk_ani_result* join,
                         sk_derep_stats* stats, sk_store_stats* store_stats) {
  return dereplicate_store_impl(WHO_STORE, ctxs, n_ctx, st, mp, rank, 0, dp, device_budget, rep, cluster, join, stats, store_stats);
}

int sk_dereplicate_store_fixed(sk_ctx* const* ctxs, uint32_t n_ctx, const sk_sketch_store* st, const sk_map_params* mp,
                               const uint32_t* rank, uint32_t n_fixed, const sk_derep_params* dp, uint64_t device_budget,
                               uint32_t* rep, uint32_t* cluster, sk_ani_result* join, sk_derep_stats* stats, sk_store_stats* store_stats) {
  return dereplicate_store_impl("sk_dereplicate_store_fixed", ctxs, n_ctx, st, mp, rank, n_fixed, dp, device_budget, rep, cluster, join,
                                stats, store_stats);
}
