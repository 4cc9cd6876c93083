// store.cu -- the triangle beyond one GPU's memory: a host-resident sketch store and working-set chaining.
//
// sk_sketch_store keeps every genome's sketch (the 12 blob arrays of sk_internal.h, k-mer hash table included) as one
// contiguous record in pinned, device-mapped host slabs of a fixed size.  Adding a set packs it into a device blob with its
// tables and scatters the blob's per-genome slices into their records with ONE batched device memcpy whose destinations are
// mapped host memory.  Gathering is the mirror image: ONE batched memcpy whose sources are the records of the listed genomes
// pulls them over PCIe straight into a device blob in the layout sk_sketch_set_unpack reads (no host-side copy, no staging
// buffer), and the existing unpack builds the set without rebuilding the tables.
// sk_triangle_store screens the markers of every genome, plans working sets (ws_plan.hpp) and lets one host thread per
// context gather and chain them in plan order (chain_working_sets, store_ws.hpp).  sk_query_ref_store does the same for every
// (reference, query) pair of two stores: one marker screen of all references against all queries, working sets that each hold
// some references and some queries, gathered from their own stores.  Both keep the rows with ani > 0.1.
#include <algorithm>
#include <cstdlib>
#include <string>
#include <vector>

#include "sk_internal.h"
#include "store_ws.hpp"
#include "ws_plan.hpp"

using namespace sk;

struct sk_sketch_store {
  sk_sketch_params sp{};
  struct Slab { uint8_t* host = nullptr; uint8_t* dev = nullptr; size_t size = 0, used = 0; };
  std::vector<Slab> slabs;
  size_t slab_bytes = 1ull << 30;
  struct Genome {
    uint32_t slab = 0;
    uint64_t off = 0;                   // record offset inside the slab
    uint64_t n[N_COUNTS] = {};          // S U M C HT
    uint64_t total_len = 0;
    uint64_t ctg0 = 0;                  // first contig length in ctg_len
    uint64_t slice[BLOB_ARRAYS] = {};   // slice offsets inside the record
  };
  std::vector<Genome> g;
  std::vector<uint32_t> ctg_len;
  std::vector<uint64_t> name_rank;
};

namespace {

// The working sets of plan chained on the contexts (chain_working_sets), keeping ani > 0.1 (src/triangle.rs:99,
// src/dist.rs:115,139): the kept rows sorted by (ref_id, query_id) as a malloc'd array, and s, holding the screen's time, with
// the working sets' counts and times in *stats
template <class Plan>
int chain_and_keep(const char* who, sk_ctx* const* ctxs, uint32_t n_ctx, const sk_sketch_store* a, const sk_sketch_store* b, const Plan& plan,
                   const sk_map_params* mp, sk_store_stats s, sk_ani_result** out, uint64_t* n_out, sk_store_stats* stats) {
  std::vector<std::vector<sk_ani_result>> kept(n_ctx);
  SK_TRY(chain_working_sets(who, ctxs, n_ctx, a, b, plan, mp, [&](uint32_t d, const auto&, const std::vector<sk_ani_result>& rows) {
    for (const sk_ani_result& r : rows) if (r.ani > 0.1f) kept[d].push_back(r);
  }, s));
  std::vector<sk_ani_result> res;
  for (const auto& k : kept) res.insert(res.end(), k.begin(), k.end());
  std::sort(res.begin(), res.end(), [](const sk_ani_result& x, const sk_ani_result& y) { return x.ref_id != y.ref_id ? x.ref_id < y.ref_id : x.query_id < y.query_id; });
  SK_TRY(hand_out(ctxs[0], res, out, n_out));
  if (stats) *stats = s;
  return SK_OK;
}

}  // namespace

extern "C" {

int sk_sketch_store_create(const sk_sketch_params* sp, sk_sketch_store** out) {
  if (!sp || !out) return SK_ERR_PARAM;
  sk_sketch_store* st = new sk_sketch_store();
  st->sp = *sp;
  if (const char* e = getenv("SK_STORE_SLAB_MB")) st->slab_bytes = std::max<size_t>(1, (size_t)atoll(e)) << 20;   // test hook: many slabs
  *out = st;
  return SK_OK;
}

int sk_sketch_store_free(sk_sketch_store* st) {
  if (!st) return SK_OK;
  for (auto& s : st->slabs) cudaFreeHost(s.host);
  delete st;
  return SK_OK;
}

uint32_t sk_sketch_store_n_genomes(const sk_sketch_store* st) { return st ? (uint32_t)st->g.size() : 0; }

uint64_t sk_sketch_store_genome_bytes(const sk_sketch_store* st, uint32_t g) {
  if (!st || g >= st->g.size()) return 0;
  return genome_bytes(st->g[g].n);
}

int sk_sketch_store_set_name_ranks(sk_sketch_store* st, const uint64_t* ranks) {
  if (!st || (!ranks && !st->g.empty())) return SK_ERR_PARAM;
  for (size_t g = 0; g < st->g.size(); g++) st->name_rank[g] = ranks[g];
  return SK_OK;
}

int sk_sketch_store_add(sk_sketch_store* st, const sk_sketch_set* set) {
  if (!st || !set) return SK_ERR_PARAM;
  sk_ctx* ctx = set->ctx;
  if (!same_params(set->sp, st->sp)) { ctx->err = "sk_sketch_store_add: the set's sketch parameters differ from the store's"; return SK_ERR_PARAM; }
  if ((uint64_t)st->g.size() + set->G >= (1ull << 32)) { ctx->err = "sk_sketch_store_add: more than 2^32 genomes"; return SK_ERR_PARAM; }
  SK_CUDA(cudaSetDevice(ctx->device));
  if (set->G == 0) return SK_OK;
  // the set's own blob with its k-mer tables
  uint64_t bytes = 0, words = 0;
  SK_TRY(sk_sketch_set_subset_blob_size(set, nullptr, 0, SK_PACK_TABLES, &bytes, &words));
  DTmp<uint8_t> blob;
  if (blob.alloc(bytes, ctx) != cudaSuccess) { ctx->err = "sk_sketch_store_add: out of device memory for the blob"; return SK_ERR_NOMEM; }
  std::vector<uint64_t> words_v(words);
  SK_TRY(sk_sketch_set_pack_subset(set, nullptr, 0, SK_PACK_TABLES, blob.p, words_v.data()));
  const SetMeta m = decode_meta(words_v.data());
  const uint32_t G = (uint32_t)m.G;
  const BlobLayout b = blob_layout(G, m.n);
  // records in the slabs (host-side bookkeeping first, so that a failed slab allocation leaves the store unchanged)
  std::vector<sk_sketch_store::Genome> add(G);
  std::vector<sk_sketch_store::Slab> new_slabs;
  auto slab_at = [&](uint32_t i) -> sk_sketch_store::Slab& { return i < st->slabs.size() ? st->slabs[i] : new_slabs[i - st->slabs.size()]; };
  uint32_t cur = st->slabs.empty() ? 0 : (uint32_t)st->slabs.size() - 1;
  std::vector<size_t> used;
  for (auto& s : st->slabs) used.push_back(s.used);
  auto fail_slabs = [&](int rc) { for (auto& s : new_slabs) cudaFreeHost(s.host); return rc; };
  for (uint32_t i = 0; i < G; i++) {
    sk_sketch_store::Genome& e = add[i];
    for (int x = 0; x < N_COUNTS; x++) e.n[x] = m.off[x][i + 1] - m.off[x][i];
    e.total_len = m.total_len[i];
    const size_t need = std::max<uint64_t>(al256(genome_slices(e.n, e.slice)), 256);
    const uint32_t n_slabs = (uint32_t)(st->slabs.size() + new_slabs.size());
    if (n_slabs == 0 || used[cur] + need > slab_at(cur).size) {
      sk_sketch_store::Slab s;
      s.size = std::max(st->slab_bytes, need);
      cudaError_t err = cudaHostAlloc((void**)&s.host, s.size, cudaHostAllocMapped | cudaHostAllocPortable);
      if (err == cudaSuccess) err = cudaHostGetDevicePointer((void**)&s.dev, s.host, 0);
      if (err != cudaSuccess) {
        cudaGetLastError();
        if (s.host) cudaFreeHost(s.host);
        ctx->err = "sk_sketch_store_add: cannot allocate " + std::to_string(s.size >> 20) + " MiB of pinned host memory: " + cudaGetErrorString(err);
        return fail_slabs(SK_ERR_NOMEM);
      }
      new_slabs.push_back(s);
      used.push_back(0);
      cur = n_slabs;
    }
    e.slab = cur; e.off = used[cur];
    used[cur] += need;
  }
  // one batched copy: blob slices -> records in mapped host memory
  SegmentCopy cp;
  cp.batched = true;
  for (uint32_t i = 0; i < G; i++)
    for (int a = 0; a < BLOB_ARRAYS; a++) {
      const ArrayDesc& d = SET_ARRAYS[a];
      cp.add(blob.p + b.off[a] + array_index(a, i, m.off[d.by][i]) * d.esz, slab_at(add[i].slab).dev + add[i].off + add[i].slice[a],
             array_elems(a, 1, add[i].n) * d.esz);
    }
  const int rc = cp.run(ctx);
  if (rc != SK_OK) return fail_slabs(rc);
  // commit
  for (auto& s : new_slabs) st->slabs.push_back(s);
  for (size_t i = 0; i < st->slabs.size(); i++) st->slabs[i].used = used[i];
  uint64_t mx = 0;
  for (uint64_t r : st->name_rank) mx = std::max(mx, r + 1);
  for (uint32_t i = 0; i < G; i++) {
    add[i].ctg0 = st->ctg_len.size();
    for (uint64_t c = m.off[CNT_C][i]; c < m.off[CNT_C][i + 1]; c++) st->ctg_len.push_back((uint32_t)m.ctg_len[c]);
    st->g.push_back(add[i]);
    st->name_rank.push_back(mx + set->name_rank[i]);
  }
  return SK_OK;
}

int sk_sketch_store_gather(sk_ctx* ctx, const sk_sketch_store* st, const uint32_t* genomes, uint32_t n, int flags, sk_sketch_set** out) {
  if (!ctx || !out) return SK_ERR_PARAM;
  *out = nullptr;
  if (!st || (n && !genomes)) { ctx->err = "sk_sketch_store_gather: NULL store or genome list"; return SK_ERR_PARAM; }
  if (flags != 0 && flags != SK_PACK_MARKERS_ONLY) { ctx->err = "sk_sketch_store_gather: flags must be 0 or SK_PACK_MARKERS_ONLY"; return SK_ERR_PARAM; }
  for (uint32_t i = 0; i < n; i++) {
    if (genomes[i] >= st->g.size()) { ctx->err = "sk_sketch_store_gather: genome " + std::to_string(genomes[i]) + " out of range"; return SK_ERR_PARAM; }
    if (i && genomes[i] <= genomes[i - 1]) { ctx->err = "sk_sketch_store_gather: genomes must be ascending without duplicates"; return SK_ERR_PARAM; }
  }
  SK_CUDA(cudaSetDevice(ctx->device));
  const bool mo = flags == SK_PACK_MARKERS_ONLY;
  // the metadata sk_sketch_set_pack_subset would write for these genomes, over the store's records
  SetMeta m;
  m.c = st->sp.c; m.k = st->sp.k; m.marker_c = st->sp.marker_c; m.tables = !mo;
  for (uint32_t i = 0; i < n; i++) {
    const sk_sketch_store::Genome& e = st->g[genomes[i]];
    meta_push(m, e.n, mo, e.total_len, st->ctg_len.begin() + e.ctg0, st->ctg_len.begin() + e.ctg0 + e.n[CNT_C]);
  }
  const BlobLayout b = blob_layout(n, m.n);
  DTmp<uint8_t> blob;
  if (blob.alloc(b.total, ctx) != cudaSuccess) { ctx->err = "sk_sketch_store_gather: out of device memory (" + std::to_string(b.total >> 20) + " MiB blob)"; return SK_ERR_NOMEM; }
  SK_CUDA(zero_absent_arrays(ctx, blob.p, b, mo, m.tables));
  SegmentCopy cp;
  cp.batched = true;
  for (uint32_t i = 0; i < n; i++) {
    const sk_sketch_store::Genome& e = st->g[genomes[i]];
    const uint8_t* rec = st->slabs[e.slab].dev + e.off;
    for (int a = 0; a < BLOB_ARRAYS; a++) {
      const ArrayDesc& d = SET_ARRAYS[a];
      if (array_travels(a, mo, m.tables)) cp.add(rec + e.slice[a], blob.p + b.off[a] + array_index(a, i, m.off[d.by][i]) * d.esz, array_elems(a, 1, e.n) * d.esz);
    }
  }
  SK_TRY(cp.run(ctx));
  if (mo && n) SK_CUDA(cudaStreamSynchronize(ctx->stream));
  std::vector<uint64_t> meta(meta_words(n, m.n[CNT_C], m.tables));
  encode_meta(m, meta.data());
  const void* bp = blob.p;
  const uint64_t* mp = meta.data();
  SK_TRY(sk_sketch_set_unpack(ctx, 1, &bp, &mp, out));
  for (uint32_t i = 0; i < n; i++) (*out)->name_rank[i] = st->name_rank[genomes[i]];
  (*out)->ranks_user_set = true;
  return SK_OK;
}

int sk_triangle_store(sk_ctx* const* ctxs, uint32_t n_ctx, const sk_sketch_store* st, const sk_map_params* mp, uint64_t device_budget,
                      sk_ani_result** out, uint64_t* n_out, sk_store_stats* stats) {
  const char* const who = "sk_triangle_store";
  if (!ctxs || n_ctx == 0 || !ctxs[0]) return SK_ERR_PARAM;
  sk_ctx* ctx = ctxs[0];
  if (!st || !mp || !out || !n_out) { ctx->err = "sk_triangle_store: NULL argument"; return SK_ERR_PARAM; }
  *out = nullptr; *n_out = 0;
  SK_TRY(check_contexts(ctxs, n_ctx));
  const uint32_t N = (uint32_t)st->g.size();
  uint64_t budget = 0;
  SK_TRY(working_set_budget(ctxs, n_ctx, device_budget, &budget));
  std::vector<uint64_t> gbytes(N);
  for (uint32_t g = 0; g < N; g++) gbytes[g] = sk_sketch_store_genome_bytes(st, g);
  std::string perr;
  if (!skws::genomes_fit(gbytes, budget, perr)) { ctx->err = std::string(who) + ": " + perr; return SK_ERR_NOMEM; }
  // ---- 1. screen: markers of every genome on context 0
  sk_store_stats s{};
  const double t0 = now_s();
  std::vector<uint64_t> pairs;
  {
    SK_CUDA(cudaSetDevice(ctx->device));
    sk_sketch_set* mk = nullptr;
    SK_TRY(gather_markers(ctx, st, &mk));
    uint64_t* p = nullptr; uint64_t np = 0;
    const int rc = sk_screen_triangle(ctx, mk, mp, &p, &np);
    sk_sketch_set_free(mk);
    SK_TRY(rc);
    pairs.assign(p, p + np);
    sk_free(p);
  }
  s.t_screen = now_s() - t0;
  // ---- 2. plan
  skws::Plan plan;
  if (!skws::plan_working_sets(pairs, gbytes, budget, plan, perr)) { ctx->err = std::string(who) + ": " + perr; return SK_ERR_NOMEM; }
  // ---- 3. contexts take the working sets in plan order
  return chain_and_keep(who, ctxs, n_ctx, st, st, plan, mp, s, out, n_out, stats);
}

int sk_query_ref_store(sk_ctx* const* ctxs, uint32_t n_ctx, const sk_sketch_store* refs, const sk_sketch_store* queries, const sk_map_params* mp,
                       int mode, uint64_t device_budget, sk_ani_result** out, uint64_t* n_out, sk_store_stats* stats) {
  const char* const who = "sk_query_ref_store";
  if (!ctxs || n_ctx == 0 || !ctxs[0]) return SK_ERR_PARAM;
  sk_ctx* ctx = ctxs[0];
  if (!refs || !queries || !mp || !out || !n_out) { ctx->err = "sk_query_ref_store: NULL argument"; return SK_ERR_PARAM; }
  *out = nullptr; *n_out = 0;
  if (mode < 0 || mode > 3) { ctx->err = "sk_query_ref_store: mode " + std::to_string(mode) + " is not 0-3"; return SK_ERR_PARAM; }
  if (!same_params(refs->sp, queries->sp)) { ctx->err = "sk_query_ref_store: the stores' sketch parameters differ"; return SK_ERR_PARAM; }
  SK_TRY(check_contexts(ctxs, n_ctx));
  const uint32_t NR = (uint32_t)refs->g.size(), NQ = (uint32_t)queries->g.size();
  uint64_t budget = 0;
  SK_TRY(working_set_budget(ctxs, n_ctx, device_budget, &budget));
  std::vector<uint64_t> rbytes(NR), qbytes(NQ);
  for (uint32_t g = 0; g < NR; g++) rbytes[g] = sk_sketch_store_genome_bytes(refs, g);
  for (uint32_t g = 0; g < NQ; g++) qbytes[g] = sk_sketch_store_genome_bytes(queries, g);
  std::string perr;   // split point NR: every genome of rbytes is a reference, and with split point 0 every one of qbytes a query
  if (!skws::genomes_fit(rbytes, budget, perr, NR) || !skws::genomes_fit(qbytes, budget, perr, 0)) {
    ctx->err = std::string(who) + ": " + perr;
    return SK_ERR_NOMEM;
  }
  // ---- 1. screen: markers of every reference and every query on context 0
  sk_store_stats s{};
  const double t0 = now_s();
  std::vector<uint64_t> pairs;
  if (NR && NQ) {
    SK_CUDA(cudaSetDevice(ctx->device));
    sk_sketch_set *rm = nullptr, *qm = nullptr;
    int rc = gather_markers(ctx, refs, &rm);
    if (rc == SK_OK) rc = gather_markers(ctx, queries, &qm);
    uint64_t* p = nullptr; uint64_t np = 0;
    if (rc == SK_OK) rc = sk_screen_query_ref(ctx, rm, qm, mp, mode, &p, &np);
    if (rm) sk_sketch_set_free(rm);
    if (qm) sk_sketch_set_free(qm);
    SK_TRY(rc);
    pairs.assign(p, p + np);    // sorted (r << 32 | q)
    sk_free(p);
  }
  s.t_screen = now_s() - t0;
  // ---- 2. plan
  skws::QrPlan plan;
  if (!skws::plan_query_ref_working_sets(pairs, rbytes, qbytes, budget, plan, perr)) { ctx->err = std::string(who) + ": " + perr; return SK_ERR_NOMEM; }
  // ---- 3. contexts take the working sets in plan order: gather the references and the queries, chain
  return chain_and_keep(who, ctxs, n_ctx, refs, queries, plan, mp, s, out, n_out, stats);
}

}  // extern "C"
