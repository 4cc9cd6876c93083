// api.cu -- C ABI glue of libskani_b200.so: context, sketch-set lifecycle, host->device staging.
#include <sched.h>

#include <cub/cub.cuh>

#include <algorithm>
#include <chrono>
#include <cmath>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <functional>
#include <thread>

#include "host_pack.hpp"
#include "sk_core.cuh"
#include "sk_internal.h"

using namespace sk;

// ---- SkArena ------------------------------------------------------------------------------------------------
cudaError_t SkArena::alloc(void** out, size_t bytes) {
  std::lock_guard<std::mutex> lk(mu);
  const size_t need = (std::max<size_t>(bytes, 1) + 511) & ~(size_t)511;
  for (int pass = 0; pass < 2; pass++) {
    for (size_t si = 0; si < slabs.size(); si++) {
      auto& fb = slabs[si].free_blocks;
      for (auto it = fb.begin(); it != fb.end(); ++it) {
        if (it->second >= need) {
          const size_t off = it->first, sz = it->second;
          fb.erase(it);
          if (sz > need) fb[off + need] = sz - need;
          void* p = slabs[si].base + off;
          live[p] = {(int)si, need};
          *out = p;
          return cudaSuccess;
        }
      }
    }
    if (pass == 1) break;
    // grow: a new slab, geometrically sized
    size_t slab = std::max<size_t>(need, std::min<size_t>(16ull << 30, std::max<size_t>(1ull << 30, total)));
    uint8_t* base = nullptr;
    cudaError_t e = cudaMalloc((void**)&base, slab);
    if (e != cudaSuccess && slab > need) { cudaGetLastError(); slab = need; e = cudaMalloc((void**)&base, slab); }
    if (e != cudaSuccess) return e;
    Slab s; s.base = base; s.size = slab; s.free_blocks[0] = slab;
    slabs.push_back(std::move(s));
    total += slab;
  }
  return cudaErrorMemoryAllocation;
}
void SkArena::release(void* p) {
  if (!p) return;
  std::lock_guard<std::mutex> lk(mu);
  auto it = live.find(p);
  if (it == live.end()) return;
  const int si = it->second.first;
  size_t sz = it->second.second;
  live.erase(it);
  auto& fb = slabs[si].free_blocks;
  size_t off = (uint8_t*)p - slabs[si].base;
  auto nx = fb.lower_bound(off);
  if (nx != fb.end() && off + sz == nx->first) { sz += nx->second; nx = fb.erase(nx); }     // coalesce with the next block
  if (nx != fb.begin()) {
    auto pv = std::prev(nx);
    if (pv->first + pv->second == off) { off = pv->first; sz += pv->second; fb.erase(pv); }  // and with the previous one
  }
  fb[off] = sz;
}
void SkArena::destroy() {
  std::lock_guard<std::mutex> lk(mu);
  for (auto& s : slabs) cudaFree(s.base);
  slabs.clear(); live.clear(); total = 0;
}

// ---- SkPool ---------------------------------------------------------------------------------------------------
SkPool::SkPool(int n_threads) {
  for (int t = 1; t < n_threads; t++)
    th.emplace_back([this] {
      uint64_t seen = 0;
      for (;;) {
        const std::function<void(size_t)>* f;
        size_t n;
        {
          std::unique_lock<std::mutex> lk(mu);
          cv.wait(lk, [&] { return stop || gen != seen; });
          if (stop) return;
          seen = gen; f = fn; n = n_tasks;
        }
        for (size_t i; (i = next.fetch_add(1)) < n;) (*f)(i);
        { std::lock_guard<std::mutex> lk(mu); if (--working == 0) cv_done.notify_all(); }
      }
    });
}
SkPool::~SkPool() {
  { std::lock_guard<std::mutex> lk(mu); stop = true; }
  cv.notify_all();
  for (auto& t : th) t.join();
}
void SkPool::run(size_t n, const std::function<void(size_t)>& f) {
  if (n == 0) return;
  if (th.empty() || n == 1) { for (size_t i = 0; i < n; i++) f(i); return; }
  { std::lock_guard<std::mutex> lk(mu); fn = &f; n_tasks = n; next.store(0); working = th.size(); gen++; }
  cv.notify_all();
  for (size_t i; (i = next.fetch_add(1)) < n;) f(i);
  std::unique_lock<std::mutex> lk(mu);
  cv_done.wait(lk, [&] { return working == 0; });
}

namespace sk {
// host threads this context may use for packing: the CPUs the process can run on, capped by the container's CPU quota,
// divided among the ranks of one box (torchrun's LOCAL_WORLD_SIZE) / the contexts of one process; SK_PACK_THREADS overrides
static int host_pack_threads(const sk_ctx* ctx) {
  if (const char* e = getenv("SK_PACK_THREADS")) return std::max(1, atoi(e));
  int n = (int)std::thread::hardware_concurrency();
  cpu_set_t cs;
  if (sched_getaffinity(0, sizeof(cs), &cs) == 0) n = CPU_COUNT(&cs);
  if (FILE* f = fopen("/sys/fs/cgroup/cpu.max", "r")) {
    char q[64] = {0};
    long per = 0;
    if (fscanf(f, "%63s %ld", q, &per) == 2 && strcmp(q, "max") != 0 && per > 0) n = std::min(n, (int)std::ceil(atof(q) / (double)per));
    fclose(f);
  }
  int share = std::max(1, ctx->cpu_share);
  if (const char* e = getenv("LOCAL_WORLD_SIZE")) share *= std::max(1, atoi(e));
  return std::max(1, std::min(64, n / share - 1));
}
SkPool* ctx_pool(sk_ctx* ctx) {
  if (!ctx->pool) ctx->pool = new SkPool(host_pack_threads(ctx));
  return ctx->pool;
}

// ---- sk_sketch_set_import_batch: device-side (contig, pos) ordering of imported records --------------------------------
__global__ void import_keys_kernel(const uint64_t* __restrict__ rec_off, const uint32_t* __restrict__ pos, const uint32_t* __restrict__ cc,
                                   uint64_t* __restrict__ keys, uint32_t* __restrict__ vals) {
  const uint32_t g = blockIdx.x;
  const uint64_t b = rec_off[g], e = rec_off[g + 1];
  for (uint64_t i = b + (uint64_t)blockIdx.y * blockDim.x + threadIdx.x; i < e; i += (uint64_t)blockDim.x * gridDim.y) {
    keys[i] = ((uint64_t)(cc[i] >> 1) << 32) | pos[i];
    vals[i] = (uint32_t)(i - b);
  }
}
__global__ void import_gather_kernel(const uint64_t* __restrict__ rec_off, const uint32_t* __restrict__ perm, const uint32_t* __restrict__ k,
                                     const uint32_t* __restrict__ p, const uint32_t* __restrict__ c, uint32_t* __restrict__ ok,
                                     uint32_t* __restrict__ op, uint32_t* __restrict__ oc) {
  const uint32_t g = blockIdx.x;
  const uint64_t b = rec_off[g], e = rec_off[g + 1];
  for (uint64_t i = b + (uint64_t)blockIdx.y * blockDim.x + threadIdx.x; i < e; i += (uint64_t)blockDim.x * gridDim.y) {
    const uint64_t src = b + perm[i];
    ok[i] = k[src]; op[i] = p[src]; oc[i] = c[src];
  }
}
// per contig (+ one sentinel per genome): local index of its first record = lower bound of (contig << 32) in the genome's sorted keys
__global__ void import_ctab_kernel(const uint64_t* __restrict__ rec_off, const uint64_t* __restrict__ ctg_off, uint32_t G,
                                   const uint64_t* __restrict__ skeys, uint32_t* __restrict__ ctab, uint32_t* __restrict__ bad) {
  const uint64_t t = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;      // entry index in [0, C + G)
  const uint64_t total = ctg_off[G] + G;
  if (t >= total) return;
  uint32_t lo = 0, hi = G;                                                 // genome g with ctg_off[g] + g <= t < ctg_off[g + 1] + g + 1
  while (hi - lo > 1) { const uint32_t m = (lo + hi) >> 1; if (ctg_off[m] + m <= t) lo = m; else hi = m; }
  const uint32_t g = lo;
  const uint32_t c = (uint32_t)(t - ctg_off[g] - g), nc = (uint32_t)(ctg_off[g + 1] - ctg_off[g]);
  const uint64_t b = rec_off[g], e = rec_off[g + 1];
  uint64_t a = b, z = e;
  const uint64_t want = (uint64_t)c << 32;
  while (a < z) { const uint64_t m = (a + z) >> 1; if (skeys[m] < want) a = m + 1; else z = m; }
  ctab[t] = (uint32_t)(a - b);
  if (c == nc && a != e) atomicOr(bad, 1u);                                // a record names a contig the sketch does not have
}

// flags `bad` when some v[i] >= limit.  Imported markers must be < 2^42 and seed k-mers < 4^k: the views build their sort
// keys as (genome << 42 | marker) and (genome << 2k | k-mer), so a larger value would land in another genome's list.
template <typename T>
__global__ void import_range_kernel(const T* __restrict__ v, uint64_t n, uint64_t limit, uint32_t* __restrict__ bad, uint32_t flag) {
  bool over = false;
  for (uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (uint64_t)blockDim.x * gridDim.x) over |= (uint64_t)v[i] >= limit;
  if (over) atomicOr(bad, flag);
}

__global__ void stage_copy_kernel(uint32_t* __restrict__ dst, const uint32_t* __restrict__ src, size_t n_words) {
  size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n_words) dst[i] = src[i];
}
// host -> device upload of a small parameter block, ordered on ctx->stream, without touching the H2D copy engine
cudaError_t h2d_small(sk_ctx* ctx, void* dst, const void* src, size_t bytes) {
  if (bytes == 0) return cudaSuccess;
  const size_t CAP = 64ull << 20;
  if ((bytes & 3) || ((uintptr_t)dst & 3) || bytes > CAP / 4) return cudaMemcpyAsync(dst, src, bytes, cudaMemcpyHostToDevice, ctx->stream);
  if (!ctx->stage) {
    cudaError_t e = cudaHostAlloc((void**)&ctx->stage, CAP, cudaHostAllocMapped | cudaHostAllocPortable);
    if (e != cudaSuccess) return e;
    ctx->stage_cap = CAP; ctx->stage_pos = 0;
  }
  size_t pos = (ctx->stage_pos + 15) & ~(size_t)15;
  if (pos + bytes > ctx->stage_cap) {          // ring wrap: everything queued so far must have been consumed
    cudaError_t e = cudaStreamSynchronize(ctx->stream);
    if (e != cudaSuccess) return e;
    pos = 0;
  }
  memcpy(ctx->stage + pos, src, bytes);
  const size_t nw = bytes / 4;
  stage_copy_kernel<<<(unsigned)((nw + 255) / 256), 256, 0, ctx->stream>>>((uint32_t*)dst, (const uint32_t*)(ctx->stage + pos), nw);
  ctx->stage_pos = pos + bytes;
  return cudaGetLastError();
}
}  // namespace sk

namespace {
constexpr size_t SUBBATCH_MAX = 2048ull << 20;  // bases per seeding sub-batch: bounds the per-base temporaries ...
constexpr size_t SUBBATCH_MIN = 256ull << 20;   // ... while keeping >= ~8 sub-batches so H2D copies overlap the kernels
inline size_t subbatch_bytes(uint64_t total) { return std::min<size_t>(SUBBATCH_MAX, std::max<size_t>(SUBBATCH_MIN, total / 8)); }

int check_sketch_params(sk_ctx* ctx, const sk_sketch_params* sp) {
  if (!sp || sp->c == 0 || sp->marker_c == 0 || sp->k == 0) { ctx->err = "bad sketch params"; return SK_ERR_PARAM; }
  if (sp->c > sp->marker_c) { ctx->err = "c > marker_c is not allowed (src/params.rs:183-185)"; return SK_ERR_PARAM; }
  if (sp->k > 16) { ctx->err = "k > 16 is not allowed (src/seeding.rs:239-241)"; return SK_ERR_PARAM; }
  return SK_OK;
}

void parallel_memcpy(sk_ctx* ctx, void* dst, const void* src, size_t n) {
  if (n < (8u << 20)) { memcpy(dst, src, n); return; }
  const size_t chunk = 4u << 20, nt = (n + chunk - 1) / chunk;
  ctx_pool(ctx)->run(nt, [&](size_t t) { const size_t b = t * chunk; memcpy((uint8_t*)dst + b, (const uint8_t*)src + b, std::min(chunk, n - b)); });
}

template <typename T>
int concat_dev(sk_ctx* ctx, const std::vector<const T*>& parts, const std::vector<size_t>& counts, T** out) {
  size_t total = 0;
  for (size_t c : counts) total += c;
  T* p = nullptr;
  SK_CUDA(ctx->arena.alloc((void**)&p, std::max<size_t>(total, 1) * sizeof(T)));
  size_t o = 0;
  for (size_t i = 0; i < parts.size(); i++) {
    if (counts[i]) SK_CUDA(cudaMemcpyAsync(p + o, parts[i], counts[i] * sizeof(T), cudaMemcpyDeviceToDevice, ctx->stream));
    o += counts[i];
  }
  *out = p;
  return SK_OK;
}

// concatenate sketch sets (genome-local indexing everywhere, so only the prefix offsets shift).  with_tables: the parts
// carry their k-mer hash tables (ht_off / htab) and the result takes them over by copy instead of rebuilding them.
int concat_sets(sk_ctx* ctx, const std::vector<const sk_sketch_set*>& parts, sk_sketch_set** out, bool with_tables = false) {
  sk_sketch_set* s = new sk_sketch_set();
  s->ctx = ctx;
  s->sp = parts.empty() ? sk_sketch_params{125, 15, 1000} : parts[0]->sp;
  struct Guard { sk_sketch_set* s; ~Guard() { if (s) { free_set_device(s); delete s; } } } guard{s};
  s->seed_off = {0}; s->uk_off = {0}; s->mk_off = {0}; s->ctg_off = {0};
  std::vector<size_t> nS, nU, nM, nC, nUG, nCG, nB;
  for (auto* p : parts) {
    if (p->sp.c != s->sp.c || p->sp.k != s->sp.k || p->sp.marker_c != s->sp.marker_c) { ctx->err = "sketch parameter mismatch"; return SK_ERR_PARAM; }
    for (uint32_t g = 0; g < p->G; g++) {
      s->seed_off.push_back(s->seed_off.back() + (p->seed_off[g + 1] - p->seed_off[g]));
      s->uk_off.push_back(s->uk_off.back() + (p->uk_off[g + 1] - p->uk_off[g]));
      s->mk_off.push_back(s->mk_off.back() + (p->mk_off[g + 1] - p->mk_off[g]));
      s->ctg_off.push_back(s->ctg_off.back() + (p->ctg_off[g + 1] - p->ctg_off[g]));
      s->total_len.push_back(p->total_len[g]);
      s->name_rank.push_back(s->G + g);
    }
    s->ctg_len.insert(s->ctg_len.end(), p->ctg_len.begin(), p->ctg_len.end());
    s->G += p->G;
    nS.push_back(p->S); nU.push_back(p->U); nM.push_back(p->M); nC.push_back(p->C);
    nUG.push_back(p->U + p->G); nCG.push_back(p->C + p->G); nB.push_back((size_t)p->G * (UBUCKETS + 1));
  }
  s->S = s->seed_off.back(); s->U = s->uk_off.back(); s->M = s->mk_off.back(); s->C = s->ctg_off.back();
#define CAT(field, T, counts)                                         \
  {                                                                   \
    std::vector<const T*> v;                                          \
    for (auto* p : parts) v.push_back(p->field);                      \
    SK_TRY(concat_dev<T>(ctx, v, counts, &s->field));                 \
  }
  CAT(pv_kmer, uint32_t, nS) CAT(pv_pos, uint32_t, nS) CAT(pv_cc, uint32_t, nS) CAT(pv_mult, uint16_t, nS)
  CAT(kv_pos, uint32_t, nS) CAT(kv_cc, uint32_t, nS) CAT(ukmer, uint32_t, nU) CAT(ustart, uint32_t, nUG)
  CAT(markers, uint64_t, nM) CAT(ctg_rec_off, uint32_t, nCG) CAT(d_ctg_len, uint32_t, nC)
  if (with_tables) {
    std::vector<size_t> nH;
    s->ht_off = {0};
    for (auto* p : parts) {
      for (uint32_t g = 0; g < p->G; g++) s->ht_off.push_back(s->ht_off.back() + (p->ht_off[g + 1] - p->ht_off[g]));
      nH.push_back(p->ht_off[p->G]);
    }
    CAT(htab, unsigned long long, nH)
  }
#undef CAT
  SK_CUDA(cudaStreamSynchronize(ctx->stream));
  guard.s = nullptr;
  *out = s;
  return SK_OK;
}
}  // namespace

extern "C" {

// low_priority: the worker context of the pipelined sk_triangle.  Its chaining kernels share the GPU with the producer's
// seeding kernels; the producer is on the critical path (upload -> seed must keep pace with PCIe), the chains only have to be
// done by the end, so the producer's stream gets the higher hardware priority (its blocks are scheduled first)
static int ctx_create_impl(int device, sk_ctx** out, bool low_priority) {
  if (!out) return SK_ERR_PARAM;
  *out = nullptr;
  int ndev = 0;
  if (cudaGetDeviceCount(&ndev) != cudaSuccess || ndev == 0 || device < 0 || device >= ndev) return SK_ERR_CUDA;  // no CPU fallback
  if (cudaSetDevice(device) != cudaSuccess) return SK_ERR_CUDA;
  sk_ctx* ctx = new sk_ctx();
  ctx->device = device;
  cudaDeviceProp prop;
  if (cudaGetDeviceProperties(&prop, device) != cudaSuccess) { delete ctx; return SK_ERR_CUDA; }
  ctx->sm_count = prop.multiProcessorCount;
  int prio_least = 0, prio_greatest = 0;
  if (cudaDeviceGetStreamPriorityRange(&prio_least, &prio_greatest) != cudaSuccess) { prio_least = prio_greatest = 0; cudaGetLastError(); }
  if (cudaStreamCreateWithPriority(&ctx->stream, cudaStreamNonBlocking, low_priority ? prio_least : prio_greatest) != cudaSuccess ||
      cudaStreamCreateWithFlags(&ctx->copy_stream, cudaStreamNonBlocking) != cudaSuccess) { delete ctx; return SK_ERR_CUDA; }
  for (int i = 0; i < 2; i++) {
    cudaEventCreateWithFlags(&ctx->pinned_free[i], cudaEventDisableTiming);
    cudaEventCreateWithFlags(&ctx->h2d_done[i], cudaEventDisableTiming);
  }
  // keep freed stream-ordered allocations cached in the pool
  cudaMemPool_t pool;
  if (cudaDeviceGetDefaultMemPool(&pool, device) == cudaSuccess) {
    uint64_t thr = ~0ull;
    cudaMemPoolSetAttribute(pool, cudaMemPoolAttrReleaseThreshold, &thr);
  }
  *out = ctx;
  return SK_OK;
}

int sk_ctx_create(int device, sk_ctx** out) { return ctx_create_impl(device, out, false); }
int sk_ctx_create_worker(int device, sk_ctx** out) { return ctx_create_impl(device, out, true); }   // internal (triangle.cu)

int sk_ctx_destroy(sk_ctx* ctx) {
  if (!ctx) return SK_OK;
  cudaSetDevice(ctx->device);
  cudaStreamSynchronize(ctx->stream);
  if (ctx->child) { sk_ctx_destroy(ctx->child); ctx->child = nullptr; }
  if (ctx->chain_scratch && ctx->chain_scratch_free) ctx->chain_scratch_free(ctx->chain_scratch);
  if (ctx->pool) { delete ctx->pool; ctx->pool = nullptr; }
  for (int i = 0; i < 2; i++) {
    if (ctx->dbuf[i]) cudaFree(ctx->dbuf[i]);
    if (ctx->dP[i]) cudaFree(ctx->dP[i]);
    if (ctx->dNM[i]) cudaFree(ctx->dNM[i]);
    if (ctx->hP[i]) cudaFreeHost(ctx->hP[i]);
    if (ctx->hNM[i]) cudaFreeHost(ctx->hNM[i]);
    if (ctx->x0[i]) cudaEventDestroy(ctx->x0[i]);
    if (ctx->x1[i]) cudaEventDestroy(ctx->x1[i]);
  }
  ctx->arena.destroy();
  if (ctx->stage) cudaFreeHost(ctx->stage);
  for (auto& b : ctx->mbox_blocks) cudaFreeHost(b.first);
  for (int i = 0; i < 2; i++) {
    if (ctx->pinned[i]) cudaFreeHost(ctx->pinned[i]);
    if (ctx->pinned_free[i]) cudaEventDestroy(ctx->pinned_free[i]);
    if (ctx->h2d_done[i]) cudaEventDestroy(ctx->h2d_done[i]);
  }
  cudaStreamDestroy(ctx->stream);
  cudaStreamDestroy(ctx->copy_stream);
  delete ctx;
  return SK_OK;
}

int sk_device_count(void) {
  int n = 0;
  if (cudaGetDeviceCount(&n) != cudaSuccess) { cudaGetLastError(); return 0; }
  return n;
}

int sk_device_memory(int device, uint64_t* free_bytes, uint64_t* total_bytes) {
  if (!free_bytes || !total_bytes || device < 0 || device >= sk_device_count()) return SK_ERR_PARAM;
  int prev = 0;
  size_t f = 0, t = 0;
  if (cudaGetDevice(&prev) != cudaSuccess || cudaSetDevice(device) != cudaSuccess) { cudaGetLastError(); return SK_ERR_CUDA; }
  const cudaError_t e = cudaMemGetInfo(&f, &t);
  cudaSetDevice(prev);
  if (e != cudaSuccess) { cudaGetLastError(); return SK_ERR_CUDA; }
  *free_bytes = f; *total_bytes = t;
  return SK_OK;
}

int sk_ctx_set_seeding_semantics(sk_ctx* ctx, int semantics) {
  if (!ctx || (semantics != SK_SEED_AVX2 && semantics != SK_SEED_SCALAR)) return SK_ERR_PARAM;
  ctx->seed_scalar = semantics == SK_SEED_SCALAR;
  if (ctx->child) ctx->child->seed_scalar = ctx->seed_scalar;
  return SK_OK;
}

const char* sk_last_error(const sk_ctx* ctx) { return ctx ? ctx->err.c_str() : "null context"; }
uint64_t sk_ctx_launch_count(const sk_ctx* ctx) { return ctx ? ctx->launches + (ctx->child ? ctx->child->launches : 0) : 0; }   // incl. the pipelined triangle's worker context
void* sk_ctx_stream(const sk_ctx* ctx) { return ctx ? (void*)ctx->stream : nullptr; }
void sk_free(void* p) { free(p); }

int sk_ctx_set_timing(sk_ctx* ctx, int on) {
  if (!ctx) return SK_ERR_PARAM;
  ctx->timing = on != 0;
  return SK_OK;
}

// "name total_ms launches\n" per kernel, accumulated since the last call with reset != 0
int sk_ctx_get_timing(sk_ctx* ctx, char* buf, uint64_t cap, int reset) {
  if (!ctx || !buf || cap == 0) return SK_ERR_PARAM;
  SK_CUDA(cudaSetDevice(ctx->device));
  SK_CUDA(cudaStreamSynchronize(ctx->stream));
  for (auto& p : ctx->pending) {
    float ms = 0;
    if (cudaEventElapsedTime(&ms, p.e0, p.e1) == cudaSuccess) {
      auto& a = ctx->timing_acc[p.name];
      a.first += ms; a.second += 1;
    }
    cudaEventDestroy(p.e0); cudaEventDestroy(p.e1);
  }
  ctx->pending.clear();
  std::string out;
  for (auto& kv : ctx->timing_acc) out += kv.first + " " + std::to_string(kv.second.first) + " " + std::to_string(kv.second.second) + "\n";
  if (out.size() + 1 > cap) return SK_ERR_NOMEM;
  memcpy(buf, out.c_str(), out.size() + 1);
  if (reset) ctx->timing_acc.clear();
  return SK_OK;
}

int sk_sketch_set_free(sk_sketch_set* set) {
  if (!set) return SK_OK;
  cudaSetDevice(set->ctx->device);
  free_set_device(set);
  delete set;
  return SK_OK;
}

uint32_t sk_sketch_set_n_genomes(const sk_sketch_set* set) { return set ? set->G : 0; }

int sk_sketch_set_genome_info(const sk_sketch_set* s, uint32_t g, uint64_t* n_records, uint64_t* n_kmers,
                              uint64_t* n_markers, uint64_t* n_contigs, uint64_t* total_len) {
  if (!s || g >= s->G) return SK_ERR_PARAM;
  if (n_records) *n_records = s->seed_off[g + 1] - s->seed_off[g];
  if (n_kmers) *n_kmers = s->uk_off[g + 1] - s->uk_off[g];
  if (n_markers) *n_markers = s->mk_off[g + 1] - s->mk_off[g];
  if (n_contigs) *n_contigs = s->ctg_off[g + 1] - s->ctg_off[g];
  if (total_len) *total_len = s->total_len[g];
  return SK_OK;
}

int sk_sketch_set_export(const sk_sketch_set* s, uint32_t g, uint32_t* kmer, uint32_t* pos, uint32_t* contig_canon,
                         uint64_t* markers, uint32_t* contig_lengths) {
  if (!s || g >= s->G) return SK_ERR_PARAM;
  sk_ctx* ctx = s->ctx;
  SK_CUDA(cudaSetDevice(ctx->device));
  size_t b = s->seed_off[g], n = s->seed_off[g + 1] - b;
  if (pos && n) SK_CUDA(cudaMemcpy(pos, s->kv_pos + b, n * 4, cudaMemcpyDeviceToHost));
  if (contig_canon && n) SK_CUDA(cudaMemcpy(contig_canon, s->kv_cc + b, n * 4, cudaMemcpyDeviceToHost));
  if (kmer && n) {
    size_t ub = s->uk_off[g], un = s->uk_off[g + 1] - ub;
    std::vector<uint32_t> uk(un), us(un + 1);
    SK_CUDA(cudaMemcpy(uk.data(), s->ukmer + ub, un * 4, cudaMemcpyDeviceToHost));
    SK_CUDA(cudaMemcpy(us.data(), s->ustart + ub + g, (un + 1) * 4, cudaMemcpyDeviceToHost));
    for (size_t u = 0; u < un; u++)
      for (uint32_t i = us[u]; i < us[u + 1]; i++) kmer[i] = uk[u];
  }
  size_t mb = s->mk_off[g], mn = s->mk_off[g + 1] - mb;
  if (markers && mn) SK_CUDA(cudaMemcpy(markers, s->markers + mb, mn * 8, cudaMemcpyDeviceToHost));
  if (contig_lengths) {
    size_t cb = s->ctg_off[g], cn = s->ctg_off[g + 1] - cb;
    for (size_t i = 0; i < cn; i++) contig_lengths[i] = s->ctg_len[cb + i];
  }
  return SK_OK;
}

int sk_sketch_set_set_name_ranks(sk_sketch_set* set, const uint64_t* ranks) {
  if (!set || !ranks) return SK_ERR_PARAM;
  for (uint32_t g = 0; g < set->G; g++) set->name_rank[g] = ranks[g];
  set->ranks_user_set = true;
  return SK_OK;
}

int sk_sketch_set_append(sk_sketch_set* dst, const sk_sketch_set* src) {
  if (!dst || !src) return SK_ERR_PARAM;
  sk_ctx* ctx = dst->ctx;
  SK_CUDA(cudaSetDevice(ctx->device));
  sk_sketch_set* merged = nullptr;
  SK_TRY(concat_sets(ctx, {dst, src}, &merged));
  struct MG { sk_sketch_set* s; ~MG() { if (s) { free_set_device(s); delete s; } } } mg{merged};
  SK_TRY(build_hash(ctx, merged));
  mg.s = nullptr;
  const bool user_ranks = dst->ranks_user_set || src->ranks_user_set;
  free_set_device(dst);
  std::vector<uint64_t> ranks = dst->name_rank;
  uint64_t mx = 0;
  for (uint64_t r : ranks) mx = std::max(mx, r + 1);
  for (uint64_t r : src->name_rank) ranks.push_back(mx + r);
  *dst = *merged;  // takes over device pointers + metadata
  dst->name_rank = ranks;
  dst->ranks_user_set = user_ranks;
  merged->pv_kmer = nullptr;  // ownership moved
  delete merged;
  return SK_OK;
}

namespace {
inline const void* set_array(const sk_sketch_set* s, int i) {
  const void* p[BLOB_ARRAYS] = {s->pv_kmer, s->pv_pos, s->pv_cc, s->pv_mult, s->kv_pos, s->kv_cc, s->ukmer, s->ustart, s->markers, s->ctg_rec_off,
                                 s->d_ctg_len, s->htab};
  return p[i];
}
}  // namespace

int sk_sketch_set_blob_size(const sk_sketch_set* s, uint64_t* device_bytes, uint64_t* host_meta_words) {
  if (!s || !device_bytes || !host_meta_words) return SK_ERR_PARAM;
  *device_bytes = blob_layout(s->G, s->S, s->U, s->M, s->C).total;
  *host_meta_words = meta_words(s->G, s->C, false);
  return SK_OK;
}

int sk_sketch_set_pack(const sk_sketch_set* s, void* d_blob, uint64_t* meta) {
  if (!s || !d_blob || !meta) return SK_ERR_PARAM;
  sk_ctx* ctx = s->ctx;
  SK_CUDA(cudaSetDevice(ctx->device));
  BlobLayout b = blob_layout(s->G, s->S, s->U, s->M, s->C);
  for (int i = 0; i < 11; i++)
    if (b.bytes[i]) SK_CUDA(cudaMemcpyAsync((uint8_t*)d_blob + b.off[i], set_array(s, i), b.bytes[i], cudaMemcpyDeviceToDevice, ctx->stream));
  uint64_t* m = meta;
  *m++ = s->G; *m++ = s->S; *m++ = s->U; *m++ = s->M; *m++ = s->C; *m++ = s->sp.c; *m++ = s->sp.k; *m++ = s->sp.marker_c; *m++ = 0; *m++ = 0;
  for (uint32_t g = 0; g <= s->G; g++) *m++ = s->seed_off[g];
  for (uint32_t g = 0; g <= s->G; g++) *m++ = s->uk_off[g];
  for (uint32_t g = 0; g <= s->G; g++) *m++ = s->mk_off[g];
  for (uint32_t g = 0; g <= s->G; g++) *m++ = s->ctg_off[g];
  for (uint32_t g = 0; g < s->G; g++) *m++ = s->total_len[g];
  for (size_t c = 0; c < s->C; c++) *m++ = s->ctg_len[c];
  SK_CUDA(cudaStreamSynchronize(ctx->stream));
  return SK_OK;
}

namespace {
// host-side plan of a subset blob: maximal runs of consecutive genomes are copied with one memcpy per array
struct SubsetPlan {
  std::vector<uint32_t> idx;                        // selected genomes, in output order
  std::vector<uint64_t> seed_off, uk_off, mk_off, ctg_off, ht_off;
  size_t S = 0, U = 0, M = 0, C = 0, HT = 0;
  bool tables = false;
};
int plan_subset(const sk_sketch_set* s, const uint32_t* genomes, uint32_t n, int flags, SubsetPlan& pl) {
  const bool mo = (flags & SK_PACK_MARKERS_ONLY) != 0;
  if (!genomes) { n = s->G; pl.idx.resize(n); for (uint32_t i = 0; i < n; i++) pl.idx[i] = i; }
  else pl.idx.assign(genomes, genomes + n);
  pl.seed_off.assign(n + 1, 0); pl.uk_off.assign(n + 1, 0); pl.mk_off.assign(n + 1, 0); pl.ctg_off.assign(n + 1, 0); pl.ht_off.assign(n + 1, 0);
  pl.tables = !mo && (flags & SK_PACK_TABLES) != 0 && s->htab != nullptr && s->ht_off.size() == (size_t)s->G + 1;
  for (uint32_t i = 0; i < n; i++) {
    const uint32_t g = pl.idx[i];
    if (g >= s->G) { s->ctx->err = "subset genome index out of range"; return SK_ERR_PARAM; }
    pl.ht_off[i + 1] = pl.ht_off[i] + (pl.tables ? s->ht_off[g + 1] - s->ht_off[g] : 0);
    pl.seed_off[i + 1] = pl.seed_off[i] + (mo ? 0 : s->seed_off[g + 1] - s->seed_off[g]);
    pl.uk_off[i + 1] = pl.uk_off[i] + (mo ? 0 : s->uk_off[g + 1] - s->uk_off[g]);
    pl.ctg_off[i + 1] = pl.ctg_off[i] + (mo ? 0 : s->ctg_off[g + 1] - s->ctg_off[g]);
    pl.mk_off[i + 1] = pl.mk_off[i] + (s->mk_off[g + 1] - s->mk_off[g]);
  }
  pl.S = pl.seed_off[n]; pl.U = pl.uk_off[n]; pl.M = pl.mk_off[n]; pl.C = pl.ctg_off[n]; pl.HT = pl.ht_off[n];
  return SK_OK;
}
}  // namespace

int sk_sketch_set_subset_blob_size(const sk_sketch_set* s, const uint32_t* genomes, uint32_t n, int flags, uint64_t* device_bytes,
                                   uint64_t* host_meta_words) {
  if (!s || !device_bytes || !host_meta_words) return SK_ERR_PARAM;
  SubsetPlan pl;
  SK_TRY(plan_subset(s, genomes, n, flags, pl));
  const size_t G = pl.idx.size();
  *device_bytes = blob_layout(G, pl.S, pl.U, pl.M, pl.C, pl.HT).total;
  *host_meta_words = meta_words(G, pl.C, pl.tables);
  return SK_OK;
}

int sk_sketch_set_pack_subset(const sk_sketch_set* s, const uint32_t* genomes, uint32_t n, int flags, void* d_blob, uint64_t* meta) {
  if (!s || !d_blob || !meta) return SK_ERR_PARAM;
  sk_ctx* ctx = s->ctx;
  SK_CUDA(cudaSetDevice(ctx->device));
  SubsetPlan pl;
  SK_TRY(plan_subset(s, genomes, n, flags, pl));
  const bool mo = (flags & SK_PACK_MARKERS_ONLY) != 0;
  const uint32_t G = (uint32_t)pl.idx.size();
  const BlobLayout b = blob_layout(G, pl.S, pl.U, pl.M, pl.C, pl.HT);
  uint8_t* base = (uint8_t*)d_blob;
  cudaStream_t st = ctx->stream;
  // A scattered subset (the cross-block fetch of a genome order unrelated to relatedness asks for thousands of separate runs,
  // 12 arrays each) would cost tens of thousands of cudaMemcpyAsync calls (150 ms measured for 5 000 genomes): beyond a few
  // runs the segments are collected and copied by ONE batched device memcpy (cub::DeviceMemcpy::Batched).
  uint32_t n_runs = 0;
  for (uint32_t i = 0; i < G;) { uint32_t j = i + 1; while (j < G && pl.idx[j] == pl.idx[j - 1] + 1) j++; n_runs++; i = j; }
  const bool batched = n_runs > 8;
  std::vector<const void*> seg_src;
  std::vector<void*> seg_dst;
  std::vector<size_t> seg_n;
  auto cp = [&](int arr, size_t dst_elem, const void* src, size_t src_elem, size_t count, size_t esz) -> cudaError_t {
    if (count == 0) return cudaSuccess;
    if (batched) {
      seg_src.push_back((const uint8_t*)src + src_elem * esz); seg_dst.push_back(base + b.off[arr] + dst_elem * esz); seg_n.push_back(count * esz);
      return cudaSuccess;
    }
    return cudaMemcpyAsync(base + b.off[arr] + dst_elem * esz, (const uint8_t*)src + src_elem * esz, count * esz, cudaMemcpyDeviceToDevice, st);
  };
  if (mo) {   // one zero sentinel per genome in the group-start and contig-record tables
    if (G) SK_CUDA(cudaMemsetAsync(base + b.off[7], 0, (size_t)G * 4, st));
    if (G) SK_CUDA(cudaMemsetAsync(base + b.off[9], 0, (size_t)G * 4, st));
  }
  for (uint32_t i = 0; i < G;) {
    uint32_t j = i + 1;
    while (j < G && pl.idx[j] == pl.idx[j - 1] + 1) j++;       // run [i, j) = source genomes [a, e)
    const uint32_t a = pl.idx[i], e = pl.idx[j - 1] + 1;
    if (!mo) {
      const size_t so = s->seed_off[a], ns = s->seed_off[e] - so, uo = s->uk_off[a], nu = s->uk_off[e] - uo;
      const size_t co = s->ctg_off[a], nc = s->ctg_off[e] - co;
      SK_CUDA(cp(0, pl.seed_off[i], s->pv_kmer, so, ns, 4)); SK_CUDA(cp(1, pl.seed_off[i], s->pv_pos, so, ns, 4));
      SK_CUDA(cp(2, pl.seed_off[i], s->pv_cc, so, ns, 4));   SK_CUDA(cp(3, pl.seed_off[i], s->pv_mult, so, ns, 2));
      SK_CUDA(cp(4, pl.seed_off[i], s->kv_pos, so, ns, 4));  SK_CUDA(cp(5, pl.seed_off[i], s->kv_cc, so, ns, 4));
      SK_CUDA(cp(6, pl.uk_off[i], s->ukmer, uo, nu, 4));
      SK_CUDA(cp(7, pl.uk_off[i] + i, s->ustart, uo + a, nu + (e - a), 4));          // + one sentinel per genome
      SK_CUDA(cp(9, pl.ctg_off[i] + i, s->ctg_rec_off, co + a, nc + (e - a), 4));
      SK_CUDA(cp(10, pl.ctg_off[i], s->d_ctg_len, co, nc, 4));
      if (pl.tables) SK_CUDA(cp(11, pl.ht_off[i], s->htab, s->ht_off[a], s->ht_off[e] - s->ht_off[a], 8));
    }
    SK_CUDA(cp(8, pl.mk_off[i], s->markers, s->mk_off[a], s->mk_off[e] - s->mk_off[a], 8));
    i = j;
  }
  if (batched && !seg_n.empty()) {
    const size_t ns = seg_n.size();
    DTmp<const void*> d_src; DTmp<void*> d_dst; DTmp<size_t> d_n;
    SK_CUDA(d_src.alloc(ns, ctx)); SK_CUDA(d_dst.alloc(ns, ctx)); SK_CUDA(d_n.alloc(ns, ctx));
    SK_CUDA(cudaMemcpyAsync(d_src.p, seg_src.data(), ns * sizeof(void*), cudaMemcpyHostToDevice, st));
    SK_CUDA(cudaMemcpyAsync(d_dst.p, seg_dst.data(), ns * sizeof(void*), cudaMemcpyHostToDevice, st));
    SK_CUDA(cudaMemcpyAsync(d_n.p, seg_n.data(), ns * sizeof(size_t), cudaMemcpyHostToDevice, st));
    size_t tb = 0;
    SK_CUDA(cub::DeviceMemcpy::Batched(nullptr, tb, d_src.p, d_dst.p, d_n.p, (uint32_t)ns, st));
    DTmp<uint8_t> tmp;
    SK_CUDA(tmp.alloc(tb, ctx));
    SK_CUDA(cub::DeviceMemcpy::Batched(tmp.p, tb, d_src.p, d_dst.p, d_n.p, (uint32_t)ns, st));
    sk::count_launch(ctx);
    SK_CUDA(cudaStreamSynchronize(st));      // the host-side segment lists and the temporaries are released below
  }
  uint64_t* m = meta;
  *m++ = G; *m++ = pl.S; *m++ = pl.U; *m++ = pl.M; *m++ = pl.C; *m++ = s->sp.c; *m++ = s->sp.k; *m++ = s->sp.marker_c;
  *m++ = pl.HT; *m++ = pl.tables ? 1 : 0;
  for (uint32_t g = 0; g <= G; g++) *m++ = pl.seed_off[g];
  for (uint32_t g = 0; g <= G; g++) *m++ = pl.uk_off[g];
  for (uint32_t g = 0; g <= G; g++) *m++ = pl.mk_off[g];
  for (uint32_t g = 0; g <= G; g++) *m++ = pl.ctg_off[g];
  for (uint32_t g = 0; g < G; g++) *m++ = s->total_len[pl.idx[g]];
  if (!mo)
    for (uint32_t g = 0; g < G; g++)
      for (uint64_t c = s->ctg_off[pl.idx[g]]; c < s->ctg_off[pl.idx[g] + 1]; c++) *m++ = s->ctg_len[c];
  if (pl.tables) for (uint32_t g = 0; g <= G; g++) *m++ = pl.ht_off[g];
  SK_CUDA(cudaStreamSynchronize(st));
  return SK_OK;
}

int sk_sketch_set_unpack(sk_ctx* ctx, uint32_t n_parts, const void* const* d_blobs, const uint64_t* const* metas, sk_sketch_set** out) {
  if (!ctx || !out || n_parts == 0 || !d_blobs || !metas) return SK_ERR_PARAM;
  SK_CUDA(cudaSetDevice(ctx->device));
  // non-owning views over the blobs, then one concatenating copy
  bool all_tables = true;
  std::vector<sk_sketch_set> views(n_parts);
  std::vector<const sk_sketch_set*> vp;
  for (uint32_t i = 0; i < n_parts; i++) {
    const uint64_t* m = metas[i];
    sk_sketch_set& v = views[i];
    v.ctx = ctx;
    v.G = (uint32_t)m[0]; v.S = m[1]; v.U = m[2]; v.M = m[3]; v.C = m[4];
    v.sp.c = (uint32_t)m[5]; v.sp.k = (uint32_t)m[6]; v.sp.marker_c = (uint32_t)m[7];
    const uint64_t HT = m[8];
    const bool tables = m[9] != 0;
    all_tables = all_tables && (tables || v.U == 0);
    m += META_HEADER;
    v.seed_off.assign(m, m + v.G + 1); m += v.G + 1;
    v.uk_off.assign(m, m + v.G + 1); m += v.G + 1;
    v.mk_off.assign(m, m + v.G + 1); m += v.G + 1;
    v.ctg_off.assign(m, m + v.G + 1); m += v.G + 1;
    v.total_len.assign(m, m + v.G); m += v.G;
    v.ctg_len.resize(v.C);
    for (size_t c = 0; c < v.C; c++) v.ctg_len[c] = (uint32_t)m[c];
    v.name_rank.resize(v.G);
    if (tables) { v.ht_off.assign(m + v.C, m + v.C + v.G + 1); }
    else v.ht_off.assign((size_t)v.G + 1, 0);
    BlobLayout b = blob_layout(v.G, v.S, v.U, v.M, v.C, HT);
    uint8_t* base = (uint8_t*)d_blobs[i];
    v.htab = (unsigned long long*)(base + b.off[11]);
    v.pv_kmer = (uint32_t*)(base + b.off[0]); v.pv_pos = (uint32_t*)(base + b.off[1]); v.pv_cc = (uint32_t*)(base + b.off[2]);
    v.pv_mult = (uint16_t*)(base + b.off[3]); v.kv_pos = (uint32_t*)(base + b.off[4]); v.kv_cc = (uint32_t*)(base + b.off[5]);
    v.ukmer = (uint32_t*)(base + b.off[6]); v.ustart = (uint32_t*)(base + b.off[7]); v.markers = (uint64_t*)(base + b.off[8]);
    v.ctg_rec_off = (uint32_t*)(base + b.off[9]); v.d_ctg_len = (uint32_t*)(base + b.off[10]);
    vp.push_back(&v);
  }
  // blobs packed with SK_PACK_TABLES bring their k-mer hash tables along: no rebuild (genomes too large for a table, which
  // use the bucket index instead, fall back to the rebuild)
  if (all_tables) {
    for (auto& v : views)
      for (uint32_t g = 0; g < v.G && all_tables; g++)
        if (v.uk_off[g + 1] > v.uk_off[g] && v.ht_off[g + 1] == v.ht_off[g]) all_tables = false;
  }
  SK_TRY(concat_sets(ctx, vp, out, all_tables));
  for (auto& v : views) v.htab = nullptr;
  if (all_tables) return SK_OK;
  return build_hash(ctx, *out);
}

int sk_sketch_batch_dev(sk_ctx* ctx, const uint8_t* d_bases, const uint64_t* contig_off, uint32_t n_contigs,
                        const uint32_t* genome_of_contig, uint32_t n_genomes, const sk_sketch_params* sp,
                        sk_sketch_set** out) {
  if (!out) return SK_ERR_PARAM;
  return sk::sketch_batch_dev_parts(ctx, d_bases, contig_off, n_contigs, genome_of_contig, n_genomes, sp, out, nullptr, 0);
}

}  // extern "C"

namespace sk {
// Sequences already resident on the device: sub-batches of whole genomes through the seeding kernels.  With on_part every
// finished sub-batch is handed over (the pipelined sk_triangle on device-resident input) instead of being concatenated into *out.
int sketch_batch_dev_parts(sk_ctx* ctx, const uint8_t* d_bases, const uint64_t* contig_off, uint32_t n_contigs,
                           const uint32_t* genome_of_contig, uint32_t n_genomes, const sk_sketch_params* sp, sk_sketch_set** out,
                           const std::function<int(sk_sketch_set*, uint32_t, uint32_t)>* on_part, size_t subbatch_override) {
  if (!ctx || (!out && !on_part) || !contig_off || (!genome_of_contig && n_contigs)) return SK_ERR_PARAM;
  SK_CUDA(cudaSetDevice(ctx->device));
  SK_TRY(check_sketch_params(ctx, sp));
  // split into sub-batches of whole genomes (bounds the per-base temporaries)
  std::vector<sk_sketch_set*> parts;
  struct Guard { std::vector<sk_sketch_set*>& v; ~Guard() { for (auto* s : v) sk_sketch_set_free(s); } } guard{parts};
  uint32_t c0 = 0;
  bool first = true;
  std::vector<uint32_t> gl;
  size_t SUBBATCH = subbatch_override ? subbatch_override : subbatch_bytes(n_contigs ? contig_off[n_contigs] - contig_off[0] : 0);
  if (const char* e = getenv("SK_SUBBATCH_BYTES")) SUBBATCH = std::max<size_t>(1, (size_t)atoll(e));   // test hook: many small sub-batches
  while (c0 < n_contigs) {
    uint32_t g0 = genome_of_contig[c0];
    uint32_t c1 = c0;
    uint64_t bytes = 0;
    while (c1 < n_contigs) {
      // extend by one whole genome at a time
      uint32_t g = genome_of_contig[c1];
      uint32_t c2 = c1;
      while (c2 < n_contigs && genome_of_contig[c2] == g) c2++;
      uint64_t gb = contig_off[c2] - contig_off[c1];
      if (c1 > c0 && bytes + gb > SUBBATCH) break;
      bytes += gb;
      c1 = c2;
    }
    uint32_t g_next = (c1 < n_contigs) ? genome_of_contig[c1] : n_genomes;
    // genomes g0 .. g_next-1 belong to this part (empty genomes between are kept as empty sketches; those skipped between
    // the previous part and g0 were attributed to the previous part)
    uint32_t g_begin = first ? 0 : g0;
    first = false;
    gl.resize(c1 - c0);
    for (uint32_t i = c0; i < c1; i++) gl[i - c0] = genome_of_contig[i] - g_begin;
    sk_sketch_set* part = nullptr;
    SeedSrc src; src.d_ascii = d_bases;
    SK_TRY(sketch_batch_device(ctx, src, contig_off + c0, c1 - c0, gl.data(), g_next - g_begin, sp, &part));
    if (on_part) SK_TRY((*on_part)(part, g_begin, g_next));     // ownership moves to the callee
    else parts.push_back(part);
    c0 = c1;
  }
  if (on_part) return SK_OK;
  if (parts.empty()) {  // no contigs at all: n_genomes empty sketches
    sk_sketch_set* part = nullptr;
    uint64_t z = 0;
    SeedSrc src; src.d_ascii = d_bases;
    SK_TRY(sketch_batch_device(ctx, src, contig_off ? contig_off : &z, 0, nullptr, n_genomes, sp, &part));
    SK_TRY(build_hash(ctx, part));
    *out = part;
    return SK_OK;
  }
  if (parts.size() == 1) {
    SK_TRY(build_hash(ctx, parts[0]));
    *out = parts[0];
    parts.clear();
    return SK_OK;
  }
  std::vector<const sk_sketch_set*> cp(parts.begin(), parts.end());
  SK_TRY(concat_sets(ctx, cp, out));
  SK_TRY(build_hash(ctx, *out));
  return SK_OK;
}

static double wall_s() { return std::chrono::duration<double>(std::chrono::steady_clock::now().time_since_epoch()).count(); }

// Host -> device seeding pipeline behind sk_sketch_batch / sk_sketch_batch_2bit / sk_triangle.
//
// The input is cut into sub-batches of whole genomes.  Three stages run concurrently on double-buffered slots:
//   pack    (stager thread + the context's worker pool) a leading share of the sub-batch's contigs is converted to 2-bit
//           units + N mask on the HOST (host_pack.hpp) into pinned staging: 0.25 B/base on the wire instead of 1
//   upload  (copy stream) packed units -> dP/dNM, the remaining contigs as ASCII -> dbuf; N-mask words travel only for
//           contigs that contain 'N', the others get a device memset
//   seed    (caller thread, context stream) pack_kernel for the ASCII share + the seeding kernels (seeding.cu)
// The packed share adapts to the measured packing and PCIe rates so that packing and upload take equally long:
//   t_pack = f B / Rp  ==  t_up = B (1 - 0.75 f) / Rx   =>   f = Rp / (Rx + 0.75 Rp)        (clamped to [0, 1])
// SK_HOST_PACK=<fraction> pins the share (0 = everything as ASCII, 1 = everything packed on the host); tests use it.
// When on_part is set every finished sub-batch (a sketch set of the genomes [g_begin, g_end), without hash tables) is
// handed over as soon as it is ready and nothing is concatenated (*out stays null): the pipelined sk_triangle.
int sketch_batch_host(sk_ctx* ctx, const HostSeq& seq, const uint64_t* contig_off, uint32_t n_contigs,
                      const uint32_t* genome_of_contig, uint32_t n_genomes, const sk_sketch_params* sp, sk_sketch_set** out,
                      const std::function<int(sk_sketch_set*, uint32_t, uint32_t)>* on_part, size_t subbatch_override) {
  if (!ctx || (!out && !on_part) || !contig_off || (!genome_of_contig && n_contigs)) return SK_ERR_PARAM;
  SK_CUDA(cudaSetDevice(ctx->device));
  SK_TRY(check_sketch_params(ctx, sp));
  const bool prepacked = seq.units != nullptr;
  if (!prepacked && !seq.ascii && n_contigs && contig_off[n_contigs] > contig_off[0]) { ctx->err = "null sequence buffer"; return SK_ERR_PARAM; }
  auto is_pinned = [](const void* p) {
    if (!p) return false;
    cudaPointerAttributes attr;
    const bool pin = cudaPointerGetAttributes(&attr, p) == cudaSuccess && attr.type == cudaMemoryTypeHost;
    cudaGetLastError();
    return pin;
  };
  // is the caller's buffer page-locked? then DMA straight from it; otherwise stage through our pinned buffers
  const bool pinned_src = prepacked ? (is_pinned(seq.units) && (!seq.nmask || is_pinned(seq.nmask))) : is_pinned(seq.ascii);
  // sub-batch plan (whole genomes) + unit offset of every contig in the caller's packed layout
  struct Part { uint32_t c0, c1, g_begin, g_end; uint64_t b0, b1, units; };
  std::vector<Part> plan;
  std::vector<uint64_t> gunit(prepacked ? (size_t)n_contigs + 1 : 0, 0);
  if (prepacked) for (uint32_t i = 0; i < n_contigs; i++) gunit[i + 1] = gunit[i] + (contig_off[i + 1] - contig_off[i] + 31) / 32;
  uint32_t c0 = 0;
  uint64_t max_bytes = 0, max_units = 0;
  size_t SUBBATCH = subbatch_override ? subbatch_override : subbatch_bytes(n_contigs ? contig_off[n_contigs] - contig_off[0] : 0);
  if (const char* e = getenv("SK_SUBBATCH_BYTES")) SUBBATCH = std::max<size_t>(1, (size_t)atoll(e));   // test hook: many small sub-batches
  // large sub-batches amortise the per-sub-batch launches and host synchronisations (which cost most when the GPU is shared with
  // the chaining worker), but nothing can be seeded before the first one is packed and uploaded:
  // the first two are a quarter and a half of the size
  const bool ramp = (n_contigs ? contig_off[n_contigs] - contig_off[0] : 0) >= 4 * (uint64_t)SUBBATCH && getenv("SK_SUBBATCH_NO_RAMP") == nullptr;
  while (c0 < n_contigs) {
    uint32_t c1 = c0;
    uint64_t bytes = 0;
    // ... and towards the end every sub-batch takes half of what is left (down to an eighth of the size): what remains to be
    // seeded and chained after the LAST upload is small (the tail of the pipelined triangle)
    const uint64_t left_bytes = contig_off[n_contigs] - contig_off[c0];
    const uint64_t limit = !ramp ? SUBBATCH : plan.empty() ? SUBBATCH / 4 : plan.size() == 1 ? SUBBATCH / 2
                           : std::min<uint64_t>(SUBBATCH, std::max<uint64_t>(SUBBATCH / 8, left_bytes / 2));
    while (c1 < n_contigs) {
      uint32_t g = genome_of_contig[c1], c2 = c1;
      while (c2 < n_contigs && genome_of_contig[c2] == g) c2++;
      uint64_t gb = contig_off[c2] - contig_off[c1];
      if (c1 > c0 && bytes + gb > limit) break;
      bytes += gb;
      c1 = c2;
    }
    Part p;
    p.c0 = c0; p.c1 = c1;
    p.g_begin = plan.empty() ? 0 : genome_of_contig[c0];
    p.g_end = (c1 < n_contigs) ? genome_of_contig[c1] : n_genomes;
    p.b0 = contig_off[c0]; p.b1 = contig_off[c1];
    p.units = 0;
    for (uint32_t i = c0; i < c1; i++) {
      if (contig_off[i + 1] < contig_off[i]) { ctx->err = "contig offsets must be non-decreasing"; return SK_ERR_PARAM; }
      p.units += (contig_off[i + 1] - contig_off[i] + 31) / 32;
    }
    max_bytes = std::max(max_bytes, p.b1 - p.b0);
    max_units = std::max(max_units, p.units);
    plan.push_back(p);
    c0 = c1;
  }
  if (plan.empty()) return sk_sketch_batch_dev(ctx, nullptr, contig_off, 0, genome_of_contig, n_genomes, sp, out);
  if (max_units >= (1ull << 31)) { ctx->err = "sub-batch too large (>= 2^31 units)"; return SK_ERR_PARAM; }
  // ---- pinned share: fixed by SK_HOST_PACK, else adaptive
  double fixed_share = -1.0;
  if (const char* e = getenv("SK_HOST_PACK")) fixed_share = std::min(1.0, std::max(0.0, atof(e)));
  if (prepacked) fixed_share = 1.0;
  else if (ctx->seed_scalar) fixed_share = 0.0;   // the scalar seeder also breaks on 'n': only the device packer flags it
  SkPool* pool = ctx_pool(ctx);
  // ---- buffers (grow-only, kept in the context)
  const bool want_ascii = !prepacked && fixed_share < 1.0;
  if (want_ascii && ctx->dbuf_bytes < max_bytes + 64) {
    for (int i = 0; i < 2; i++) {
      if (ctx->dbuf[i]) SK_CUDA(cudaFree(ctx->dbuf[i]));
      ctx->dbuf[i] = nullptr;
      SK_CUDA(cudaMalloc((void**)&ctx->dbuf[i], max_bytes + 64));
    }
    ctx->dbuf_bytes = max_bytes + 64;
  }
  if (ctx->dunits < max_units) {
    for (int i = 0; i < 2; i++) {
      if (ctx->dP[i]) SK_CUDA(cudaFree(ctx->dP[i]));
      if (ctx->dNM[i]) SK_CUDA(cudaFree(ctx->dNM[i]));
      ctx->dP[i] = nullptr; ctx->dNM[i] = nullptr;
      SK_CUDA(cudaMalloc((void**)&ctx->dP[i], (max_units + 8) * 8));
      SK_CUDA(cudaMalloc((void**)&ctx->dNM[i], (max_units + 8) * 4));
    }
    ctx->dunits = max_units;
  }
  const bool need_hstage = !(prepacked && pinned_src) && fixed_share != 0.0;
  if (need_hstage && ctx->hunits < max_units) {
    for (int i = 0; i < 2; i++) {
      if (ctx->hP[i]) cudaFreeHost(ctx->hP[i]);
      if (ctx->hNM[i]) cudaFreeHost(ctx->hNM[i]);
      ctx->hP[i] = nullptr; ctx->hNM[i] = nullptr;
      SK_CUDA(cudaHostAlloc((void**)&ctx->hP[i], (max_units + 8) * 8, cudaHostAllocDefault));
      SK_CUDA(cudaHostAlloc((void**)&ctx->hNM[i], (max_units + 8) * 4, cudaHostAllocDefault));
    }
    ctx->hunits = max_units;
  }
  if (want_ascii && !pinned_src && ctx->pinned_bytes < max_bytes) {
    for (int i = 0; i < 2; i++) {
      if (ctx->pinned[i]) cudaFreeHost(ctx->pinned[i]);
      ctx->pinned[i] = nullptr;
      SK_CUDA(cudaHostAlloc((void**)&ctx->pinned[i], max_bytes, cudaHostAllocDefault));
    }
    ctx->pinned_bytes = max_bytes;
  }
  for (int i = 0; i < 2; i++) {
    if (!ctx->x0[i]) { SK_CUDA(cudaEventCreate(&ctx->x0[i])); SK_CUDA(cudaEventCreate(&ctx->x1[i])); }
  }
  if (ctx->pack_rate <= 0) ctx->pack_rate = 3.0e9 * pool->size();
  if (ctx->h2d_rate <= 0) ctx->h2d_rate = 50.0e9;

  // ---- stager thread: pack + enqueue the copies of part k; the caller seeds part k as soon as its copies are queued
  const size_t NP = plan.size();
  std::vector<uint32_t> n_packed(NP, 0);
  std::mutex mu;
  std::condition_variable cv;
  long enqueued = -1, computed = -1;
  int stager_rc = SK_OK;
  std::string stager_err;
  bool abort_all = false;
  uint64_t bases_packed = 0, bases_total = 0;
  const bool trace = getenv("SK_TRACE") != nullptr;
  const double t_call = wall_s();
  std::thread stager([&] {
    cudaSetDevice(ctx->device);
    std::vector<uint64_t> cu;           // unit offset of every contig of the part (+ total)
    std::vector<uint8_t> has_n;
    std::vector<uint64_t> xbytes(2, 0), part_bytes(2, 0);
    std::vector<double> part_pack_s(2, 0.0);
    int host_sharers = std::max(1, ctx->cpu_share);
    if (const char* ev = getenv("LOCAL_WORLD_SIZE")) host_sharers *= std::max(1, atoi(ev));
    auto fail = [&](const char* what, cudaError_t e) {
      std::lock_guard<std::mutex> lk(mu);
      stager_rc = SK_ERR_CUDA; stager_err = std::string(what) + ": " + cudaGetErrorString(e); abort_all = true;
      cv.notify_all();
    };
    for (size_t k = 0; k < NP; k++) {
      const Part& p = plan[k];
      const int b = (int)(k & 1);
      const uint32_t nc = p.c1 - p.c0;
      cudaError_t e;
      // (1) staging slot free again: the copies of part k-2 have completed; their duration gives the PCIe rate
      if (k >= 2) {
        if ((e = cudaEventSynchronize(ctx->x1[b])) != cudaSuccess) return fail("cudaEventSynchronize", e);
        float ms = 0;
        if (cudaEventElapsedTime(&ms, ctx->x0[b], ctx->x1[b]) == cudaSuccess && ms > 0.05f && xbytes[b] > (8u << 20)) {
          ctx->h2d_rate = 0.5 * ctx->h2d_rate + 0.5 * ((double)xbytes[b] / (ms * 1e-3));
          // hill climbing on the host-side stage rate of that part: input bytes / max(packing time, copy time).  Both stages
          // run concurrently and draw on the same host memory bandwidth, so balancing their measured rates (the formula below)
          // overshoots as soon as DRAM, not PCIe or the cores, is the limit (two or more GPUs per host): every second sample
          // the share moves by 0.05 in the direction that last raised the rate.
          if (fixed_share < 0 && part_bytes[b] > (64u << 20)) {
            ctx->share_acc += (double)part_bytes[b] / std::max((double)ms * 1e-3, part_pack_s[b]);
            if (++ctx->share_samples == 2) {
              const double r = ctx->share_acc / 2;
              if (ctx->share_ref_rate > 0 && r < 1.01 * ctx->share_ref_rate) ctx->share_dir = -ctx->share_dir;
              ctx->share_ref_rate = r;
              ctx->share_bias = std::min(0.5, std::max(-0.9, ctx->share_bias + 0.05 * ctx->share_dir));
              ctx->share_acc = 0; ctx->share_samples = 0;
            }
          }
        }
      }
      // (2) how many leading contigs are packed on the host
      cu.assign(nc + 1, 0);
      for (uint32_t i = 0; i < nc; i++) cu[i + 1] = cu[i] + (contig_off[p.c0 + i + 1] - contig_off[p.c0 + i] + 31) / 32;
      const uint64_t B = p.b1 - p.b0;
      // rate balance (pack time = copy time) scaled by the number of contexts that share this host's memory system as the
      // starting point, plus the correction found by the hill climber above
      double share = fixed_share >= 0 ? fixed_share : ctx->pack_rate / (ctx->h2d_rate + 0.75 * ctx->pack_rate) / (double)host_sharers + ctx->share_bias;
      share = std::min(1.0, std::max(0.0, share));
      if (fixed_share < 0 && share <= 0.0 && ctx->share_bias < 0) ctx->share_bias += 0.05;     // keep the climber inside [0, 1]
      if (fixed_share < 0 && share >= 1.0 && ctx->share_bias > 0) ctx->share_bias -= 0.05;
      uint32_t np = 0;
      if (share >= 1.0) np = nc;
      else if (share > 0.0) {
        const uint64_t target = p.b0 + (uint64_t)((double)B * share);
        while (np < nc && contig_off[p.c0 + np + 1] <= target) np++;      // whole contigs
      }
      n_packed[k] = np;
      const uint64_t pk_bases = contig_off[p.c0 + np] - p.b0, pk_units = cu[np];
      // (3) pack (or stage the caller's packed units) into the pinned slot
      has_n.assign(nc, 0);
      const uint64_t* src_units = nullptr; const uint32_t* src_nm = nullptr;
      const double tp0 = wall_s();
      if (prepacked) {
        const uint64_t u0 = gunit[p.c0];
        if (pinned_src) { src_units = seq.units + u0; src_nm = seq.nmask ? seq.nmask + u0 : nullptr; }
        else {
          parallel_memcpy(ctx, ctx->hP[b], seq.units + u0, pk_units * 8);
          if (seq.nmask) parallel_memcpy(ctx, ctx->hNM[b], seq.nmask + u0, pk_units * 4);
          src_units = ctx->hP[b]; src_nm = seq.nmask ? ctx->hNM[b] : nullptr;
        }
        if (seq.nmask) {   // which contigs carry an N at all (the others get a memset instead of a copy)
          pool->run(np, [&](size_t i) {
            const uint32_t* m = seq.nmask + u0 + cu[i];
            uint32_t any = 0;
            for (uint64_t j = 0, n = cu[i + 1] - cu[i]; j < n; j++) any |= m[j];
            has_n[i] = any != 0;
          });
        }
      } else if (np) {
        struct Task { uint32_t ci; uint64_t ub, ue; };
        std::vector<Task> tasks;
        const uint64_t TU = 32768;   // 1 Mbase per task
        for (uint32_t i = 0; i < np; i++)
          for (uint64_t ub = 0, n = cu[i + 1] - cu[i]; ub < n; ub += TU) tasks.push_back(Task{i, ub, std::min(n, ub + TU)});
        std::vector<std::atomic<uint8_t>> flag(np);
        for (auto& f : flag) f.store(0, std::memory_order_relaxed);
        uint64_t* hP = ctx->hP[b]; uint32_t* hNM = ctx->hNM[b];
        pool->run(tasks.size(), [&](size_t t) {
          const Task& tk = tasks[t];
          const uint64_t len = contig_off[p.c0 + tk.ci + 1] - contig_off[p.c0 + tk.ci];
          const uint8_t* s0 = seq.ascii + contig_off[p.c0 + tk.ci] + 32 * tk.ub;
          const uint64_t nb = std::min<uint64_t>(len - 32 * tk.ub, 32 * (tk.ue - tk.ub));
          uint64_t* P = hP + cu[tk.ci] + tk.ub;
          uint32_t* M = hNM + cu[tk.ci] + tk.ub;
          if (sk_host::pack_contig(s0, nb, P, M)) flag[tk.ci].store(1, std::memory_order_relaxed);
        });
        for (uint32_t i = 0; i < np; i++) has_n[i] = flag[i].load(std::memory_order_relaxed);
        src_units = hP; src_nm = hNM;
        const double tp = wall_s() - tp0;
        if (tp > 1e-4 && pk_bases > (8u << 20)) ctx->pack_rate = 0.5 * ctx->pack_rate + 0.5 * ((double)pk_bases / tp);
      }
      const double tp_end = wall_s();
      // staging of an unpinned ASCII tail
      const uint8_t* ascii_src = nullptr;
      const uint64_t ascii_bytes = prepacked ? 0 : (p.b1 - contig_off[p.c0 + np]);
      if (ascii_bytes) {
        if (pinned_src) ascii_src = seq.ascii + contig_off[p.c0 + np];
        else {
          if (k >= 2 && (e = cudaEventSynchronize(ctx->pinned_free[b])) != cudaSuccess) return fail("cudaEventSynchronize", e);
          parallel_memcpy(ctx, ctx->pinned[b], seq.ascii + contig_off[p.c0 + np], ascii_bytes);
          ascii_src = ctx->pinned[b];
        }
      }
      // (4) device slot free again: part k-2 has been seeded (its kernels read dP/dNM/dbuf of this slot)
      {
        std::unique_lock<std::mutex> lk(mu);
        cv.wait(lk, [&] { return abort_all || computed >= (long)k - 2; });
        if (abort_all) return;
      }
      // (5) copies
      cudaStream_t cs = ctx->copy_stream;
      uint64_t wire = 0;
      if ((e = cudaEventRecord(ctx->x0[b], cs)) != cudaSuccess) return fail("cudaEventRecord", e);
      if (pk_units) {
        if ((e = cudaMemcpyAsync(ctx->dP[b], src_units, pk_units * 8, cudaMemcpyHostToDevice, cs)) != cudaSuccess) return fail("H2D units", e);
        wire += pk_units * 8;
        for (uint32_t i = 0; i < np;) {      // runs of contigs with / without 'N'
          uint32_t j = i + 1;
          while (j < np && (has_n[j] != 0) == (has_n[i] != 0)) j++;
          const uint64_t u0 = cu[i], nu = cu[j] - cu[i];
          if (nu) {
            if (has_n[i] && src_nm) { e = cudaMemcpyAsync(ctx->dNM[b] + u0, src_nm + u0, nu * 4, cudaMemcpyHostToDevice, cs); wire += nu * 4; }
            else e = cudaMemsetAsync(ctx->dNM[b] + u0, 0, nu * 4, cs);
            if (e != cudaSuccess) return fail("H2D N mask", e);
          }
          i = j;
        }
      }
      if (ascii_bytes) {
        if ((e = cudaMemcpyAsync(ctx->dbuf[b] + (contig_off[p.c0 + np] - p.b0), ascii_src, ascii_bytes, cudaMemcpyHostToDevice, cs)) != cudaSuccess)
          return fail("H2D ASCII", e);
        wire += ascii_bytes;
        if (!pinned_src && (e = cudaEventRecord(ctx->pinned_free[b], cs)) != cudaSuccess) return fail("cudaEventRecord", e);
      }
      xbytes[b] = wire; part_bytes[b] = B; part_pack_s[b] = tp_end - tp0;
      if ((e = cudaEventRecord(ctx->x1[b], cs)) != cudaSuccess) return fail("cudaEventRecord", e);
      if ((e = cudaEventRecord(ctx->h2d_done[b], cs)) != cudaSuccess) return fail("cudaEventRecord", e);
      if (trace) fprintf(stderr, "[sk_sketch_batch] part %zu: %.0f%% of %.1f MB packed on the host (%d threads, %.1f GB/s; PCIe %.1f GB/s), %.1f MB on the wire;"
                         " pack %.1f..%.1f ms, copies queued at %.1f ms\n",
                         k, B ? 100.0 * pk_bases / B : 0.0, B / 1e6, pool->size(), ctx->pack_rate / 1e9, ctx->h2d_rate / 1e9, wire / 1e6,
                         (tp0 - t_call) * 1e3, (tp_end - t_call) * 1e3, (wall_s() - t_call) * 1e3);
      {
        std::lock_guard<std::mutex> lk(mu);
        enqueued = (long)k; bases_packed += pk_bases; bases_total += B;
      }
      cv.notify_all();
    }
  });
  struct StagerJoin {
    std::thread& t; std::mutex& mu; std::condition_variable& cv; bool& abort_all;
    ~StagerJoin() { { std::lock_guard<std::mutex> lk(mu); abort_all = true; } cv.notify_all(); if (t.joinable()) t.join(); }
  } sj{stager, mu, cv, abort_all};

  std::vector<sk_sketch_set*> parts;
  struct Guard { std::vector<sk_sketch_set*>& v; ~Guard() { for (auto* s : v) sk_sketch_set_free(s); } } guard{parts};
  std::vector<uint32_t> gl;
  for (size_t pi = 0; pi < NP; pi++) {
    const Part& p = plan[pi];
    const int b = (int)(pi & 1);
    {
      std::unique_lock<std::mutex> lk(mu);
      cv.wait(lk, [&] { return abort_all || enqueued >= (long)pi; });
      if (abort_all) { ctx->err = "staging thread: " + stager_err; return stager_rc != SK_OK ? stager_rc : SK_ERR_STATE; }
    }
    SK_CUDA(cudaStreamWaitEvent(ctx->stream, ctx->h2d_done[b], 0));
    gl.resize(p.c1 - p.c0);
    for (uint32_t i = p.c0; i < p.c1; i++) gl[i - p.c0] = genome_of_contig[i] - p.g_begin;
    SeedSrc src;
    src.d_ascii = ctx->dbuf[b]; src.ascii_base = p.b0; src.d_P = ctx->dP[b]; src.d_NM = ctx->dNM[b]; src.n_packed = n_packed[pi];
    sk_sketch_set* part = nullptr;
    const double tc0 = wall_s();
    SK_TRY(sketch_batch_device(ctx, src, contig_off + p.c0, p.c1 - p.c0, gl.data(), p.g_end - p.g_begin, sp, &part));   // ends synchronised
    if (trace) fprintf(stderr, "[sk_sketch_batch] part %zu seeded: %.1f..%.1f ms\n", pi, (tc0 - t_call) * 1e3, (wall_s() - t_call) * 1e3);
    { std::lock_guard<std::mutex> lk(mu); computed = (long)pi; }
    cv.notify_all();
    if (on_part) SK_TRY((*on_part)(part, p.g_begin, p.g_end));   // ownership moves to the callee
    else parts.push_back(part);
  }
  stager.join();
  SK_CUDA(cudaStreamSynchronize(ctx->copy_stream));
  ctx->last_pack_share = bases_total ? (double)bases_packed / (double)bases_total : 0.0;
  if (on_part) return SK_OK;
  if (parts.size() == 1) {
    SK_TRY(build_hash(ctx, parts[0]));
    *out = parts[0];
    parts.clear();
    return SK_OK;
  }
  std::vector<const sk_sketch_set*> cp(parts.begin(), parts.end());
  SK_TRY(concat_sets(ctx, cp, out));
  SK_TRY(build_hash(ctx, *out));
  return SK_OK;
}

namespace {
template <typename T>
int grow_append(sk_ctx* ctx, T** arr, size_t* cap, size_t used_alloc, size_t used, const T* src, size_t add) {
  // *cap == 0: the array was allocated at exactly `used_alloc` elements
  const size_t have = *cap ? *cap : std::max<size_t>(used_alloc, 1);
  if (used + add > have) {
    const size_t ncap = std::max<size_t>(used + add, have + have / 2);
    T* n = nullptr;
    SK_CUDA(ctx->arena.alloc((void**)&n, ncap * sizeof(T)));
    if (used) SK_CUDA(cudaMemcpyAsync(n, *arr, used * sizeof(T), cudaMemcpyDeviceToDevice, ctx->stream));
    SK_CUDA(cudaStreamSynchronize(ctx->stream));
    if (*arr) ctx->arena.release(*arr);
    *arr = n; *cap = ncap;
  }
  if (add) SK_CUDA(cudaMemcpyAsync(*arr + used, src, add * sizeof(T), cudaMemcpyDeviceToDevice, ctx->stream));
  return SK_OK;
}
}  // namespace

int append_sets_inplace(sk_ctx* ctx, sk_sketch_set** dstp, const std::vector<sk_sketch_set*>& parts, const SetReserve& hint) {
  if (parts.empty()) return SK_OK;
  sk_sketch_set* d = *dstp;
  if (!d) {   // first wave: an empty set with room for everything that is expected (estimates; arrays grow if they fall short)
    d = new sk_sketch_set();
    d->ctx = ctx; d->sp = parts[0]->sp;
    d->seed_off = {0}; d->uk_off = {0}; d->mk_off = {0}; d->ctg_off = {0}; d->ht_off = {0};
    const uint64_t S = (uint64_t)((double)hint.bases / d->sp.c * 1.06) + 64 * hint.genomes + 1024;
    const uint64_t M = (uint64_t)((double)hint.bases / d->sp.marker_c * 1.10) + 16 * hint.genomes + 1024;
    d->capS = S; d->capU = S; d->capUG = S + hint.genomes + 1; d->capM = M; d->capC = hint.contigs + 1; d->capCG = hint.contigs + hint.genomes + 1;
    d->capHT = 4 * S + 16 * hint.genomes;   // table capacity = power of two >= 2 x distinct k-mers: between 2 and 4 entries per k-mer
    struct G0 { sk_sketch_set* s; ~G0() { if (s) { free_set_device(s); delete s; } } } g0{d};
    SK_CUDA(ctx->arena.alloc((void**)&d->pv_kmer, d->capS * 4)); SK_CUDA(ctx->arena.alloc((void**)&d->pv_pos, d->capS * 4));
    SK_CUDA(ctx->arena.alloc((void**)&d->pv_cc, d->capS * 4));   SK_CUDA(ctx->arena.alloc((void**)&d->pv_mult, d->capS * 2));
    SK_CUDA(ctx->arena.alloc((void**)&d->kv_pos, d->capS * 4));  SK_CUDA(ctx->arena.alloc((void**)&d->kv_cc, d->capS * 4));
    SK_CUDA(ctx->arena.alloc((void**)&d->ukmer, d->capU * 4));   SK_CUDA(ctx->arena.alloc((void**)&d->ustart, d->capUG * 4));
    SK_CUDA(ctx->arena.alloc((void**)&d->markers, d->capM * 8)); SK_CUDA(ctx->arena.alloc((void**)&d->ctg_rec_off, d->capCG * 4));
    SK_CUDA(ctx->arena.alloc((void**)&d->d_ctg_len, d->capC * 4)); SK_CUDA(ctx->arena.alloc((void**)&d->htab, d->capHT * 8));
    g0.s = nullptr;
    *dstp = d;
  }
  const uint32_t g_begin = d->G;
  for (auto* p : parts) {
    if (p->sp.c != d->sp.c || p->sp.k != d->sp.k || p->sp.marker_c != d->sp.marker_c) { ctx->err = "sketch parameter mismatch"; return SK_ERR_PARAM; }
    size_t cS;   // the six record arrays share one capacity
    cS = d->capS; SK_TRY(grow_append(ctx, &d->pv_kmer, &cS, d->S, d->S, p->pv_kmer, p->S));
    cS = d->capS; SK_TRY(grow_append(ctx, &d->pv_pos, &cS, d->S, d->S, p->pv_pos, p->S));
    cS = d->capS; SK_TRY(grow_append(ctx, &d->pv_cc, &cS, d->S, d->S, p->pv_cc, p->S));
    cS = d->capS; SK_TRY(grow_append(ctx, &d->pv_mult, &cS, d->S, d->S, p->pv_mult, p->S));
    cS = d->capS; SK_TRY(grow_append(ctx, &d->kv_pos, &cS, d->S, d->S, p->kv_pos, p->S));
    cS = d->capS; SK_TRY(grow_append(ctx, &d->kv_cc, &cS, d->S, d->S, p->kv_cc, p->S));
    d->capS = cS;
    SK_TRY(grow_append(ctx, &d->ukmer, &d->capU, d->U, d->U, p->ukmer, p->U));
    SK_TRY(grow_append(ctx, &d->ustart, &d->capUG, d->U + d->G, d->U + d->G, p->ustart, p->U + p->G));
    SK_TRY(grow_append(ctx, &d->markers, &d->capM, d->M, d->M, p->markers, p->M));
    SK_TRY(grow_append(ctx, &d->ctg_rec_off, &d->capCG, d->C + d->G, d->C + d->G, p->ctg_rec_off, p->C + p->G));
    SK_TRY(grow_append(ctx, &d->d_ctg_len, &d->capC, d->C, d->C, p->d_ctg_len, p->C));
    for (uint32_t g = 0; g < p->G; g++) {
      d->seed_off.push_back(d->seed_off.back() + (p->seed_off[g + 1] - p->seed_off[g]));
      d->uk_off.push_back(d->uk_off.back() + (p->uk_off[g + 1] - p->uk_off[g]));
      d->mk_off.push_back(d->mk_off.back() + (p->mk_off[g + 1] - p->mk_off[g]));
      d->ctg_off.push_back(d->ctg_off.back() + (p->ctg_off[g + 1] - p->ctg_off[g]));
      d->total_len.push_back(p->total_len[g]);
      d->name_rank.push_back(d->G + g);
    }
    d->ctg_len.insert(d->ctg_len.end(), p->ctg_len.begin(), p->ctg_len.end());
    d->G += p->G; d->S += p->S; d->U += p->U; d->M += p->M; d->C += p->C;
  }
  SK_CUDA(cudaStreamSynchronize(ctx->stream));   // the parts may be released by the caller now
  return build_hash_range(ctx, d, g_begin);
}

// concatenate `parts` after `base` (may be null) into a fresh set owned by ctx, with hash tables; inputs stay valid
int merge_sets(sk_ctx* ctx, const sk_sketch_set* base, const std::vector<sk_sketch_set*>& parts, sk_sketch_set** out) {
  std::vector<const sk_sketch_set*> v;
  if (base) v.push_back(base);
  for (auto* p : parts) v.push_back(p);
  SK_TRY(concat_sets(ctx, v, out));
  return build_hash(ctx, *out);
}
}  // namespace sk

extern "C" {

int sk_sketch_batch(sk_ctx* ctx, const uint8_t* bases, const uint64_t* contig_off, uint32_t n_contigs,
                    const uint32_t* genome_of_contig, uint32_t n_genomes, const sk_sketch_params* sp, sk_sketch_set** out) {
  if (!out) return SK_ERR_PARAM;
  sk::HostSeq seq; seq.ascii = bases;
  return sk::sketch_batch_host(ctx, seq, contig_off, n_contigs, genome_of_contig, n_genomes, sp, out, nullptr, 0);
}

const char* sk_pack_impl(void) { return sk_host::pack_impl_name(); }

int sk_pack_contig(const uint8_t* ascii, uint64_t n_bases, uint64_t* units, uint32_t* nmask) {
  if ((!ascii && n_bases) || !units || !nmask) return SK_ERR_PARAM;
  sk_host::pack_contig(ascii, n_bases, units, nmask);
  return SK_OK;
}

int sk_sketch_batch_2bit(sk_ctx* ctx, const uint64_t* units, const uint32_t* nmask, const uint32_t* contig_len, uint32_t n_contigs,
                         const uint32_t* genome_of_contig, uint32_t n_genomes, const sk_sketch_params* sp, sk_sketch_set** out) {
  if (!ctx || !out || (n_contigs && (!units || !contig_len || !genome_of_contig))) return SK_ERR_PARAM;
  std::vector<uint64_t> off((size_t)n_contigs + 1, 0);
  for (uint32_t i = 0; i < n_contigs; i++) off[i + 1] = off[i] + contig_len[i];
  sk::HostSeq seq; seq.units = units; seq.nmask = nmask;
  if (n_contigs == 0 || off[n_contigs] == 0) { seq.units = nullptr; }   // nothing to stage: falls through to the empty-set path
  if (!seq.units) return sk_sketch_batch(ctx, (const uint8_t*)"", off.data(), n_contigs, genome_of_contig, n_genomes, sp, out);
  return sk::sketch_batch_host(ctx, seq, off.data(), n_contigs, genome_of_contig, n_genomes, sp, out, nullptr, 0);
}

double sk_ctx_last_pack_share(const sk_ctx* ctx) { return ctx ? ctx->last_pack_share : 0.0; }

int sk_sketch_set_import_batch(sk_ctx* ctx, const sk_sketch_params* sp, uint32_t n_genomes, const uint64_t* rec_off,
                               const uint32_t* kmer, const uint32_t* pos, const uint32_t* cc, const uint64_t* mk_off,
                               const uint64_t* markers, const uint64_t* ctg_off, const uint32_t* contig_lengths,
                               const uint64_t* total_len, sk_sketch_set** out) {
  if (!ctx || !out || n_genomes == 0 || !rec_off || !mk_off || !ctg_off) return SK_ERR_PARAM;
  const uint32_t G = n_genomes;
  const uint64_t r0 = rec_off[0], m0 = mk_off[0], c0 = ctg_off[0];
  const uint64_t n_records = rec_off[G] - r0, n_markers = mk_off[G] - m0, n_contigs = ctg_off[G] - c0;
  if ((n_records && (!kmer || !pos || !cc)) || (n_markers && !markers) || (n_contigs && !contig_lengths)) return SK_ERR_PARAM;
  SK_CUDA(cudaSetDevice(ctx->device));
  SK_TRY(check_sketch_params(ctx, sp));
  if (n_records >= (1ull << 31) || n_markers >= (1ull << 31) || n_contigs >= (1ull << 31)) {
    ctx->err = "import batch too large (>= 2^31 records, markers or contigs): import in several batches and sk_sketch_set_append";
    return SK_ERR_PARAM;
  }
  for (uint32_t g = 0; g < G; g++)
    if (rec_off[g + 1] < rec_off[g] || mk_off[g + 1] < mk_off[g] || ctg_off[g + 1] < ctg_off[g]) { ctx->err = "offsets must be non-decreasing"; return SK_ERR_PARAM; }
  sk_sketch_set* s = new sk_sketch_set();
  s->ctx = ctx; s->sp = *sp; s->G = G;
  struct Guard { sk_sketch_set* s; ~Guard() { if (s) { free_set_device(s); delete s; } } } guard{s};
  // position view = each genome's records ordered by (contig, pos); per-contig first-record table with one sentinel per
  // genome.  The records arrive in arbitrary (hash-map) order: they are sorted ON THE DEVICE (one segmented radix sort over
  // all genomes of the batch), so that a database of tens of thousands of sketches imports at PCIe speed (src/search.rs
  // deserialises and re-hashes per pair; here the host only concatenates)
  s->S = n_records; s->C = n_contigs;
  s->seed_off.resize(G + 1); s->ctg_off.resize(G + 1);
  for (uint32_t g = 0; g <= G; g++) { s->seed_off[g] = rec_off[g] - r0; s->ctg_off[g] = ctg_off[g] - c0; }
  if (n_contigs) s->ctg_len.assign(contig_lengths + c0, contig_lengths + c0 + n_contigs);
  s->total_len.resize(G);
  s->name_rank.resize(G);
  for (uint32_t g = 0; g < G; g++) {
    uint64_t tl = 0;
    if (total_len) tl = total_len[g];
    else for (uint64_t c = ctg_off[g]; c < ctg_off[g + 1]; c++) tl += contig_lengths[c];
    s->total_len[g] = tl;
    s->name_rank[g] = g;
  }
  const size_t S1 = std::max<size_t>(n_records, 1);
  SK_CUDA(ctx->arena.alloc((void**)&s->pv_kmer, S1 * 4)); SK_CUDA(ctx->arena.alloc((void**)&s->pv_pos, S1 * 4));
  SK_CUDA(ctx->arena.alloc((void**)&s->pv_cc, S1 * 4));
  SK_CUDA(ctx->arena.alloc((void**)&s->d_ctg_len, std::max<size_t>(n_contigs, 1) * 4));
  SK_CUDA(ctx->arena.alloc((void**)&s->ctg_rec_off, (size_t)(n_contigs + G + 1) * 4));
  cudaStream_t st = ctx->stream;
  SK_CUDA(cudaStreamSynchronize(st));
  if (n_contigs) SK_CUDA(cudaMemcpyAsync(s->d_ctg_len, contig_lengths + c0, n_contigs * 4, cudaMemcpyHostToDevice, st));
  DTmp<uint64_t> mraw;
  {
    DTmp<uint64_t> d_ro, d_co;
    SK_CUDA(d_ro.alloc(G + 1, ctx)); SK_CUDA(d_co.alloc(G + 1, ctx));
    SK_CUDA(h2d_small(ctx, d_ro.p, s->seed_off.data(), (G + 1) * 8));
    SK_CUDA(h2d_small(ctx, d_co.p, s->ctg_off.data(), (G + 1) * 8));
    DTmp<uint32_t> d_bad;
    SK_CUDA(d_bad.alloc(1, ctx));
    SK_CUDA(cudaMemsetAsync(d_bad.p, 0, 4, st));
    enum { BAD_CONTIG = 1, BAD_MARKER = 2, BAD_KMER = 4 };
    auto range_blocks = [](uint64_t n) { return (unsigned)std::min<uint64_t>((n + 255) / 256, 1024); };
    SK_CUDA(mraw.alloc(n_markers, ctx));
    if (n_markers) {
      SK_CUDA(cudaMemcpyAsync(mraw.p, markers + m0, n_markers * 8, cudaMemcpyHostToDevice, st));
      import_range_kernel<uint64_t><<<range_blocks(n_markers), 256, 0, st>>>(mraw.p, n_markers, 1ull << (2 * MARKER_K), d_bad.p, BAD_MARKER);
      count_launch(ctx);
    }
    if (n_records) {
      DTmp<uint32_t> rk, rp, rc, vals, perm;
      DTmp<uint64_t> keys, skeys;
      SK_CUDA(rk.alloc(n_records, ctx)); SK_CUDA(rp.alloc(n_records, ctx)); SK_CUDA(rc.alloc(n_records, ctx));
      SK_CUDA(vals.alloc(n_records, ctx)); SK_CUDA(perm.alloc(n_records, ctx)); SK_CUDA(keys.alloc(n_records, ctx)); SK_CUDA(skeys.alloc(n_records, ctx));
      SK_CUDA(cudaMemcpyAsync(rk.p, kmer + r0, n_records * 4, cudaMemcpyHostToDevice, st));
      SK_CUDA(cudaMemcpyAsync(rp.p, pos + r0, n_records * 4, cudaMemcpyHostToDevice, st));
      SK_CUDA(cudaMemcpyAsync(rc.p, cc + r0, n_records * 4, cudaMemcpyHostToDevice, st));
      if (2 * sp->k < 32) {
        import_range_kernel<uint32_t><<<range_blocks(n_records), 256, 0, st>>>(rk.p, n_records, 1ull << (2 * sp->k), d_bad.p, BAD_KMER);
        count_launch(ctx);
      }
      import_keys_kernel<<<dim3(G, 8), 256, 0, st>>>(d_ro.p, rp.p, rc.p, keys.p, vals.p); count_launch(ctx);
      size_t tb = 0;
      SK_CUDA(cub::DeviceSegmentedRadixSort::SortPairs(nullptr, tb, keys.p, skeys.p, vals.p, perm.p, (int)n_records, (int)G, d_ro.p, d_ro.p + 1, 0, 62, st));
      DTmp<uint8_t> tmp;
      SK_CUDA(tmp.alloc(tb, ctx));
      SK_CUDA(cub::DeviceSegmentedRadixSort::SortPairs(tmp.p, tb, keys.p, skeys.p, vals.p, perm.p, (int)n_records, (int)G, d_ro.p, d_ro.p + 1, 0, 62, st));
      count_launch(ctx);
      import_gather_kernel<<<dim3(G, 8), 256, 0, st>>>(d_ro.p, perm.p, rk.p, rp.p, rc.p, s->pv_kmer, s->pv_pos, s->pv_cc); count_launch(ctx);
      import_ctab_kernel<<<(unsigned)((n_contigs + G + 255) / 256), 256, 0, st>>>(d_ro.p, d_co.p, G, skeys.p, s->ctg_rec_off, d_bad.p); count_launch(ctx);
      SK_CUDA(cudaStreamSynchronize(st));
    } else {
      SK_CUDA(cudaMemsetAsync(s->ctg_rec_off, 0, (size_t)(n_contigs + G + 1) * 4, st));
    }
    uint32_t bad = 0;
    SK_CUDA(cudaMemcpyAsync(&bad, d_bad.p, 4, cudaMemcpyDeviceToHost, st));
    SK_CUDA(cudaStreamSynchronize(st));
    if (bad & BAD_MARKER) { ctx->err = "marker out of range (markers must be < 2^42)"; return SK_ERR_PARAM; }
    if (bad & BAD_KMER) { ctx->err = "seed k-mer out of range (k-mers must be < 4^k)"; return SK_ERR_PARAM; }
    if (bad & BAD_CONTIG) { ctx->err = "record contig index out of range"; return SK_ERR_PARAM; }
  }
  std::vector<uint64_t> raw_off(G + 1);
  for (uint32_t g = 0; g <= G; g++) raw_off[g] = mk_off[g] - m0;
  mbox_reset(ctx);                 // build_views takes pinned read-back space from the context's mailbox
  SK_TRY(build_views(ctx, s, mraw.p, raw_off.data()));
  SK_TRY(build_hash(ctx, s));
  SK_CUDA(cudaStreamSynchronize(ctx->stream));
  guard.s = nullptr;
  *out = s;
  return SK_OK;
}

int sk_sketch_set_import(sk_ctx* ctx, const sk_sketch_params* sp, const uint32_t* kmer, const uint32_t* pos,
                         const uint32_t* cc, uint64_t n_records, const uint64_t* markers, uint64_t n_markers,
                         const uint32_t* contig_lengths, uint32_t n_contigs, sk_sketch_set** out) {
  const uint64_t ro[2] = {0, n_records}, mo[2] = {0, n_markers}, co[2] = {0, n_contigs};
  return sk_sketch_set_import_batch(ctx, sp, 1, ro, kmer, pos, cc, mo, markers, co, contig_lengths, nullptr, out);
}

}  // extern "C"
