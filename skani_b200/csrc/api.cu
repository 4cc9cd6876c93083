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

#include "../cli/sketch_db.hpp"
#include "entry_layout.cuh"
#include "host_pack.hpp"
#include "sk_core.cuh"
#include "sk_internal.h"
#include "sketch_value.cuh"

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

// ---- sk_sketch_set_import_blobs: skani v0.3 sketch entries expanded on the device ---------------------------------------
// Blob g of a call, as the host scan (skdb::scan_entry) found it; byte offsets into the uploaded bytes, indices into the
// call's keys, multi-position lists and markers.
struct BlobDesc {
  uint64_t keys_at, key0, n_keys;      // n_keys x {u32 k-mer, u64 value}
  uint64_t list0, n_lists;             // lists [list0, list0 + n_lists) of list_at / list_len
  uint64_t markers_at, mk0, n_markers; // n_markers x u64
};
// Blobs start at arbitrary byte offsets (file-name lengths vary): loads join aligned 32-bit words with funnel shifts.
// The upload is padded so that the word after a blob's last byte exists.
__device__ __forceinline__ uint32_t load_u32_at(const uint8_t* b, uint64_t at) {
  const uint32_t* w = (const uint32_t*)(b + (at & ~3ull));
  return __funnelshift_r(w[0], w[1], (uint32_t)(at & 3) * 8);
}
__device__ __forceinline__ uint64_t load_u64_at(const uint8_t* b, uint64_t at) {
  const uint32_t* w = (const uint32_t*)(b + (at & ~3ull));
  const uint32_t sh = (uint32_t)(at & 3) * 8;
  return (uint64_t)__funnelshift_r(w[0], w[1], sh) | ((uint64_t)__funnelshift_r(w[1], w[2], sh) << 32);
}
// records per key (1, or its list's length); a multi-position index past the blob's lists names the blob in bad_blob
__global__ void blob_count_kernel(const uint8_t* __restrict__ buf, const BlobDesc* __restrict__ desc, const uint64_t* __restrict__ list_len,
                                  uint64_t* __restrict__ cnt, uint32_t* __restrict__ bad_blob) {
  const uint32_t g = blockIdx.x;
  const BlobDesc d = desc[g];
  for (uint64_t i = (uint64_t)blockIdx.y * blockDim.x + threadIdx.x; i < d.n_keys; i += (uint64_t)blockDim.x * gridDim.y) {
    const uint64_t v = load_u64_at(buf, d.keys_at + 12 * i + 4);
    uint64_t c = 1;
    if (!skdb::value_is_single(v)) {
      const uint64_t li = skdb::value_multi_index(v);
      if (li < d.n_lists) c = list_len[d.list0 + li];
      else { c = 0; atomicMin(bad_blob, g); }
    }
    cnt[d.key0 + i] = c;
  }
}
// first record of every blob (and the total): the exclusive scan of the counts at its first key
__global__ void blob_rec_off_kernel(const BlobDesc* __restrict__ desc, uint32_t G, uint64_t n_keys, const uint64_t* __restrict__ key_rec,
                                    uint64_t* __restrict__ rec_off) {
  const uint32_t g = blockIdx.x * blockDim.x + threadIdx.x;
  if (g <= G) rec_off[g] = key_rec[g < G ? desc[g].key0 : n_keys];
}
// the records in the host decoder's order (skdb::expand_records): keys in file order, each multi-position list in place
__global__ void blob_expand_kernel(const uint8_t* __restrict__ buf, const BlobDesc* __restrict__ desc, const uint64_t* __restrict__ list_at,
                                   const uint64_t* __restrict__ list_len, const uint64_t* __restrict__ key_rec, uint32_t* __restrict__ kmer,
                                   uint32_t* __restrict__ pos, uint32_t* __restrict__ cc) {
  const uint32_t g = blockIdx.x;
  const BlobDesc d = desc[g];
  for (uint64_t i = (uint64_t)blockIdx.y * blockDim.x + threadIdx.x; i < d.n_keys; i += (uint64_t)blockDim.x * gridDim.y) {
    const uint64_t at = d.keys_at + 12 * i;
    const uint32_t key = load_u32_at(buf, at);
    const uint64_t v = load_u64_at(buf, at + 4);
    const uint64_t r = key_rec[d.key0 + i];
    if (skdb::value_is_single(v)) {
      kmer[r] = key; pos[r] = skdb::value_pos(v); cc[r] = skdb::value_cc(v);
      continue;
    }
    const uint64_t li = d.list0 + skdb::value_multi_index(v), n = list_len[li], a = list_at[li];
    for (uint64_t t = 0; t < n; t++) {
      kmer[r + t] = key; pos[r + t] = load_u32_at(buf, a + 8 * t); cc[r + t] = load_u32_at(buf, a + 8 * t + 4);
    }
  }
}
__global__ void blob_markers_kernel(const uint8_t* __restrict__ buf, const BlobDesc* __restrict__ desc, uint64_t* __restrict__ mraw) {
  const uint32_t g = blockIdx.x;
  const BlobDesc d = desc[g];
  for (uint64_t i = (uint64_t)blockIdx.y * blockDim.x + threadIdx.x; i < d.n_markers; i += (uint64_t)blockDim.x * gridDim.y)
    mraw[d.mk0 + i] = load_u64_at(buf, d.markers_at + 8 * i);
}

// ---- sk_sketch_set_encode: skani v0.3 sketch entries written on the device (the inverse of the expansion above) ----------
// Entry i of a chunk, laid out by skdb::entry_layout; offsets are absolute in the chunk's device buffer.  The host writes
// the sections it owns (params, names, contig names and lengths, counts, tail) into host[host_at ...) as head | mid | tail.
struct EncDesc {
  uint64_t at, keys_at, multi_at, markers_at, mid_at, tail_at;   // entry start; first key; n_multi; first marker; mid; tail
  uint64_t host_at, head_len, mid_len, tail_len;
  uint64_t uk0, us0, rec0, mk0, f0;   // first ukmer, its ustart slot, first kv record, first marker, first key of the call
  uint64_t nu, nm, n_multi;
};
// Entries start at any byte offset (names have any length): a store is one aligned word where it can be, bytes otherwise.
__device__ __forceinline__ void store_u32_at(uint8_t* b, uint64_t at, uint32_t v) {
  if ((at & 3) == 0) { *(uint32_t*)(b + at) = v; return; }
  for (int i = 0; i < 4; i++) b[at + i] = (uint8_t)(v >> (8 * i));
}
__device__ __forceinline__ void store_u64_at(uint8_t* b, uint64_t at, uint64_t v) {
  if ((at & 7) == 0) { *(uint64_t*)(b + at) = v; return; }
  store_u32_at(b, at, (uint32_t)v);
  store_u32_at(b, at + 4, (uint32_t)(v >> 32));
}
// multi[f0 + u] = 1 when unique k-mer u of the entry has two or more records
__global__ void enc_count_kernel(const EncDesc* __restrict__ desc, const uint32_t* __restrict__ ustart, uint32_t* __restrict__ multi) {
  const EncDesc d = desc[blockIdx.x];
  for (uint64_t u = (uint64_t)blockIdx.y * blockDim.x + threadIdx.x; u < d.nu; u += (uint64_t)blockDim.x * gridDim.y)
    multi[d.f0 + u] = ustart[d.us0 + u + 1] - ustart[d.us0 + u] > 1;
}
// n_multi of every entry from the exclusive scan of the flags
__global__ void enc_n_multi_kernel(const EncDesc* __restrict__ desc, uint32_t n, const uint32_t* __restrict__ scan, uint64_t* __restrict__ n_multi) {
  const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) n_multi[i] = scan[desc[i].f0 + desc[i].nu] - scan[desc[i].f0];
}
// Key u with records kv [s, e): {k-mer, value}; a multi key's storage index is its rank r among the entry's multi keys (the
// writer's storage++ order), and its list follows the r lists before it, which hold s - u + r records.
__global__ void enc_write_kernel(const EncDesc* __restrict__ desc, const uint32_t* __restrict__ ukmer, const uint32_t* __restrict__ ustart,
                                 const uint32_t* __restrict__ kv_pos, const uint32_t* __restrict__ kv_cc, const uint64_t* __restrict__ markers,
                                 const uint32_t* __restrict__ scan, const uint8_t* __restrict__ host, uint8_t* __restrict__ out) {
  const EncDesc d = desc[blockIdx.x];
  const uint64_t t0 = (uint64_t)blockIdx.y * blockDim.x + threadIdx.x, step = (uint64_t)blockDim.x * gridDim.y;
  if (d.nu) {
    const uint32_t r0 = scan[d.f0];
    for (uint64_t u = t0; u < d.nu; u += step) {
      const uint64_t s = ustart[d.us0 + u], e = ustart[d.us0 + u + 1], at = d.keys_at + 12 * u;
      store_u32_at(out, at, ukmer[d.uk0 + u]);
      if (e - s == 1) {
        store_u64_at(out, at + 4, skdb::single_value(kv_pos[d.rec0 + s], kv_cc[d.rec0 + s]));
        continue;
      }
      const uint64_t r = scan[d.f0 + u] - r0, l = d.multi_at + 8 + 8 * r + 8 * (s - u + r);
      store_u64_at(out, at + 4, skdb::multi_value(r));
      store_u64_at(out, l, e - s);
      for (uint64_t i = s; i < e; i++) {
        store_u32_at(out, l + 8 + 8 * (i - s), kv_pos[d.rec0 + i]);
        store_u32_at(out, l + 12 + 8 * (i - s), kv_cc[d.rec0 + i]);
      }
    }
  }
  if (scan && t0 == 0) store_u64_at(out, d.multi_at, d.n_multi);
  for (uint64_t i = t0; i < d.nm; i += step) store_u64_at(out, d.markers_at + 8 * i, markers[d.mk0 + i]);
  const uint64_t nh = d.head_len + d.mid_len + d.tail_len;
  for (uint64_t i = t0; i < nh; i += step) {
    const uint64_t dst = i < d.head_len ? d.at + i : i < d.head_len + d.mid_len ? d.mid_at + (i - d.head_len) : d.tail_at + (i - d.head_len - d.mid_len);
    out[dst] = host[d.host_at + i];
  }
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

int SegmentCopy::run(sk_ctx* ctx) {
  cudaStream_t st = ctx->stream;
  const size_t ns = bytes.size();
  if (!batched) {
    for (size_t i = 0; i < ns; i++) SK_CUDA(cudaMemcpyAsync(dst[i], src[i], bytes[i], cudaMemcpyDeviceToDevice, st));
    return SK_OK;
  }
  if (ns == 0) return SK_OK;
  if (ns >= (1ull << 32)) { ctx->err = "too many copy segments"; return SK_ERR_PARAM; }
  DTmp<const void*> d_src; DTmp<void*> d_dst; DTmp<size_t> d_n;
  SK_CUDA(d_src.alloc(ns, ctx)); SK_CUDA(d_dst.alloc(ns, ctx)); SK_CUDA(d_n.alloc(ns, ctx));
  SK_CUDA(cudaMemcpyAsync(d_src.p, src.data(), ns * sizeof(void*), cudaMemcpyHostToDevice, st));
  SK_CUDA(cudaMemcpyAsync(d_dst.p, dst.data(), ns * sizeof(void*), cudaMemcpyHostToDevice, st));
  SK_CUDA(cudaMemcpyAsync(d_n.p, bytes.data(), ns * sizeof(size_t), cudaMemcpyHostToDevice, st));
  size_t tb = 0;
  auto copy = [&](void* tmp) { return cub::DeviceMemcpy::Batched(tmp, tb, d_src.p, d_dst.p, d_n.p, (uint32_t)ns, st); };
  SK_CUDA(copy(nullptr));
  DTmp<uint8_t> tmp;
  SK_CUDA(tmp.alloc(tb, ctx));
  SK_CUDA(copy(tmp.p));
  count_launch(ctx);
  SK_CUDA(cudaStreamSynchronize(st));   // the host-side lists and the temporaries are released on return
  return SK_OK;
}

cudaError_t zero_absent_arrays(sk_ctx* ctx, uint8_t* blob, const BlobLayout& b, bool markers_only, bool tables) {
  for (int a = 0; a < BLOB_ARRAYS; a++) {
    if (array_travels(a, markers_only, tables) || b.bytes[a] == 0) continue;
    const cudaError_t e = cudaMemsetAsync(blob + b.off[a], 0, b.bytes[a], ctx->stream);
    if (e != cudaSuccess) return e;
  }
  return cudaSuccess;
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

}  // namespace

namespace sk {
// is the caller's buffer page-locked? then DMA straight from it; otherwise stage through our pinned buffers
bool host_pinned(const void* p) {
  if (!p) return false;
  cudaPointerAttributes attr;
  const bool pin = cudaPointerGetAttributes(&attr, p) == cudaSuccess && attr.type == cudaMemoryTypeHost;
  cudaGetLastError();
  return pin;
}

void parallel_memcpy(sk_ctx* ctx, void* dst, const void* src, size_t n) {
  if (n < (8u << 20)) { memcpy(dst, src, n); return; }
  const size_t chunk = 4u << 20, nt = (n + chunk - 1) / chunk;
  ctx_pool(ctx)->run(nt, [&](size_t t) { const size_t b = t * chunk; memcpy((uint8_t*)dst + b, (const uint8_t*)src + b, std::min(chunk, n - b)); });
}

// host byte runs, back to back, -> dst on ctx->stream: straight from page-locked memory, otherwise staged through the
// context's two pinned buffers (one filled by the worker pool while the other is in flight)
// the context's two pinned staging buffers, at least 64 MiB each
int ensure_pinned_staging(sk_ctx* ctx) {
  const size_t CHUNK = 64ull << 20;
  if (ctx->pinned_bytes < CHUNK) {
    for (int i = 0; i < 2; i++) {
      if (ctx->pinned[i]) cudaFreeHost(ctx->pinned[i]);
      ctx->pinned[i] = nullptr;
      SK_CUDA(cudaHostAlloc((void**)&ctx->pinned[i], CHUNK, cudaHostAllocDefault));
    }
    ctx->pinned_bytes = CHUNK;
  }
  return SK_OK;
}

int upload_runs(sk_ctx* ctx, uint8_t* dst, const std::vector<std::pair<const uint8_t*, uint64_t>>& runs, bool pinned) {
  cudaStream_t st = ctx->stream;
  if (pinned) {
    for (auto& r : runs) { SK_CUDA(cudaMemcpyAsync(dst, r.first, r.second, cudaMemcpyHostToDevice, st)); dst += r.second; }
    return SK_OK;
  }
  SK_TRY(ensure_pinned_staging(ctx));
  int b = 0;
  size_t fill = 0;
  auto flush = [&]() {
    cudaError_t e = cudaMemcpyAsync(dst, ctx->pinned[b], fill, cudaMemcpyHostToDevice, st);
    if (e == cudaSuccess) e = cudaEventRecord(ctx->pinned_free[b], st);
    dst += fill; fill = 0; b ^= 1;
    return e;
  };
  for (auto& r : runs)
    for (uint64_t done = 0; done < r.second;) {
      if (fill == 0) SK_CUDA(cudaEventSynchronize(ctx->pinned_free[b]));     // the buffer's previous copy is done
      const size_t n = (size_t)std::min<uint64_t>(ctx->pinned_bytes - fill, r.second - done);
      parallel_memcpy(ctx, ctx->pinned[b] + fill, r.first + done, n);
      fill += n; done += n;
      if (fill == ctx->pinned_bytes) SK_CUDA(flush());
    }
  if (fill) SK_CUDA(flush());
  return SK_OK;
}
}  // namespace sk

namespace {

// device bytes [src, src + n) -> host dst, synchronously: straight into page-locked memory, otherwise through the context's
// two pinned buffers (the next piece in flight while the worker pool copies this one out)
int download_bytes(sk_ctx* ctx, uint8_t* dst, const uint8_t* src, uint64_t n, bool pinned) {
  cudaStream_t st = ctx->stream;
  if (pinned) {
    if (n) SK_CUDA(cudaMemcpyAsync(dst, src, n, cudaMemcpyDeviceToHost, st));
    SK_CUDA(cudaStreamSynchronize(st));
    return SK_OK;
  }
  SK_TRY(ensure_pinned_staging(ctx));
  const uint64_t P = ctx->pinned_bytes, pieces = (n + P - 1) / P;
  auto issue = [&](uint64_t k) {
    const int b = (int)(k & 1);
    cudaError_t e = cudaMemcpyAsync(ctx->pinned[b], src + k * P, std::min(P, n - k * P), cudaMemcpyDeviceToHost, st);
    return e == cudaSuccess ? cudaEventRecord(ctx->pinned_free[b], st) : e;
  };
  if (pieces) SK_CUDA(issue(0));
  for (uint64_t k = 0; k < pieces; k++) {
    if (k + 1 < pieces) SK_CUDA(issue(k + 1));     // its buffer was copied out in iteration k - 1
    SK_CUDA(cudaEventSynchronize(ctx->pinned_free[k & 1]));
    parallel_memcpy(ctx, dst + k * P, ctx->pinned[k & 1], (size_t)std::min(P, n - k * P));
  }
  SK_CUDA(cudaStreamSynchronize(st));
  return SK_OK;
}

// ---- sk_sketch_set_encode: host side.  Genomes [g0, g0 + n) of s with the caller's metadata; n_multi is filled by
// count_multi (full form) before layout() is called.
struct EncodeJob {
  const sk_sketch_set* s;
  uint32_t g0, n;
  bool full;
  const sk_entry_meta* meta;
  std::vector<EncDesc> desc;        // per entry: the set's indices; layout() adds the offsets (relative to the first entry)
  std::vector<skdb::EntryLayout> lay;
};

int check_encode_args(sk_ctx* ctx, const sk_sketch_set* s, uint32_t g0, uint32_t n, int form, const sk_entry_meta* m) {
  if (form != SK_ENTRY_FULL && form != SK_ENTRY_MARKERS) { ctx->err = "encode: unknown entry form"; return SK_ERR_PARAM; }
  if ((uint64_t)g0 + n > s->G) { ctx->err = "encode: genomes [g0, g0 + n) outside the set"; return SK_ERR_PARAM; }
  if (n == 0) return SK_OK;
  if (!m || !m->names || !m->name_off || !m->contig_first || !m->contig_order || (m->contig_first[n] > m->contig_first[0] && (!m->contig_names || !m->contig_name_off))) {
    ctx->err = "encode: metadata arrays missing"; return SK_ERR_PARAM;
  }
  for (uint32_t i = 0; i < n; i++)
    if (m->name_off[i + 1] < m->name_off[i] || m->contig_first[i + 1] < m->contig_first[i]) { ctx->err = "encode: metadata offsets decrease"; return SK_ERR_PARAM; }
  for (uint64_t j = m->contig_first[0]; j < m->contig_first[n]; j++)
    if (m->contig_name_off[j + 1] < m->contig_name_off[j]) { ctx->err = "encode: contig name offsets decrease"; return SK_ERR_PARAM; }
  return SK_OK;
}

void encode_job_init(EncodeJob& j) {
  const sk_sketch_set* s = j.s;
  j.desc.assign(j.n, EncDesc{});
  uint64_t f = 0;
  for (uint32_t i = 0; i < j.n; i++) {
    const uint32_t g = j.g0 + i;
    EncDesc& d = j.desc[i];
    d.uk0 = s->uk_off[g]; d.us0 = s->uk_off[g] + g; d.rec0 = s->seed_off[g]; d.mk0 = s->mk_off[g]; d.f0 = f;
    d.nu = j.full ? s->uk_off[g + 1] - s->uk_off[g] : 0;
    d.nm = s->mk_off[g + 1] - s->mk_off[g];
    f += d.nu;
  }
}

// the n_multi of every entry (one count pass, a scan, one copy-back); scan keeps the exclusive sum of the multi flags
int count_multi(sk_ctx* ctx, EncodeJob& j, DTmp<EncDesc>& d_desc, DTmp<uint32_t>& scan) {
  cudaStream_t st = ctx->stream;
  const uint64_t U = j.desc.back().f0 + j.desc.back().nu;
  if (U + 1 >= (1ull << 31)) { ctx->err = "encode: >= 2^31 k-mers in one call: encode fewer genomes at a time"; return SK_ERR_PARAM; }
  DTmp<uint64_t> d_nm;
  SK_CUDA(d_desc.alloc(j.n, ctx)); SK_CUDA(scan.alloc(U + 1, ctx)); SK_CUDA(d_nm.alloc(j.n, ctx));
  SK_CUDA(cudaMemcpyAsync(d_desc.p, j.desc.data(), j.n * sizeof(EncDesc), cudaMemcpyHostToDevice, st));
  SK_CUDA(cudaMemsetAsync(scan.p + U, 0, 4, st));
  if (U) { enc_count_kernel<<<dim3(j.n, 8), 256, 0, st>>>(d_desc.p, j.s->ustart, scan.p); count_launch(ctx); }
  size_t tb = 0;
  SK_CUDA(cub::DeviceScan::ExclusiveSum(nullptr, tb, scan.p, scan.p, (int)(U + 1), st));
  {
    DTmp<uint8_t> tmp;
    SK_CUDA(tmp.alloc(tb, ctx));
    SK_CUDA(cub::DeviceScan::ExclusiveSum(tmp.p, tb, scan.p, scan.p, (int)(U + 1), st));
    count_launch(ctx);
  }
  enc_n_multi_kernel<<<(j.n + 255) / 256, 256, 0, st>>>(d_desc.p, j.n, scan.p, d_nm.p); count_launch(ctx);
  std::vector<uint64_t> nm(j.n);
  SK_CUDA(cudaMemcpyAsync(nm.data(), d_nm.p, j.n * 8, cudaMemcpyDeviceToHost, st));
  SK_CUDA(cudaStreamSynchronize(st));
  for (uint32_t i = 0; i < j.n; i++) j.desc[i].n_multi = nm[i];
  return SK_OK;
}

// every entry's layout and its offset from the first entry's first byte; returns the total length
uint64_t encode_layout(EncodeJob& j) {
  const sk_sketch_set* s = j.s;
  const sk_entry_meta* m = j.meta;
  j.lay.resize(j.n);
  uint64_t at = 0;
  for (uint32_t i = 0; i < j.n; i++) {
    const uint32_t g = j.g0 + i;
    EncDesc& d = j.desc[i];
    skdb::EntryCounts c;
    c.params = c.seeds = j.full;
    c.name_len = m->name_off[i + 1] - m->name_off[i];
    c.n_keys = d.nu; c.n_multi = d.n_multi;
    c.n_records = j.full ? s->seed_off[g + 1] - s->seed_off[g] : 0;
    c.n_contigs = m->contig_first[i + 1] - m->contig_first[i];
    c.contig_name_bytes = c.n_contigs ? m->contig_name_off[m->contig_first[i + 1]] - m->contig_name_off[m->contig_first[i]] : 0;
    c.n_contig_lengths = j.full ? s->ctg_off[g + 1] - s->ctg_off[g] : 0;
    c.n_markers = d.nm;
    const skdb::EntryLayout l = skdb::entry_layout(c);
    j.lay[i] = l;
    d.at = at;
    d.keys_at = at + l.keys_at + 8; d.multi_at = at + l.multi_at; d.markers_at = at + l.markers_at + 8;
    d.mid_at = at + l.contigs_at; d.tail_at = at + l.tail_at;
    d.head_len = j.full ? l.keys_at + 8 : l.contigs_at;
    d.mid_len = l.markers_at + 8 - l.contigs_at;
    d.tail_len = skdb::TAIL_BYTES;
    at += l.length;
  }
  return at;
}

// the host sections of entry i (head | mid | tail, as put_params + put_sketch write them) appended to o
void encode_host_sections(const EncodeJob& j, uint32_t i, skdb::Out& o) {
  const sk_sketch_set* s = j.s;
  const sk_entry_meta* m = j.meta;
  const uint32_t g = j.g0 + i;
  const EncDesc& d = j.desc[i];
  auto str = [&](const char* p, uint64_t n) { o.u64(n); o.b.insert(o.b.end(), p, p + n); };
  if (j.full) {
    skdb::DiskParams dp;
    dp.c = s->sp.c; dp.k = s->sp.k; dp.marker_c = s->sp.marker_c;
    skdb::put_params(o, dp);
  }
  str(m->names + m->name_off[i], m->name_off[i + 1] - m->name_off[i]);
  o.u8(j.full ? 1 : 0);
  o.u64(d.nu);                                   // n_keys (full) or multi_position_storage's empty length (markers-only)
  o.u64(m->contig_first[i + 1] - m->contig_first[i]);
  for (uint64_t c = m->contig_first[i]; c < m->contig_first[i + 1]; c++)
    str(m->contig_names + m->contig_name_off[c], m->contig_name_off[c + 1] - m->contig_name_off[c]);
  o.u64(s->total_len[g]);
  if (j.full) {
    o.u64(s->ctg_off[g + 1] - s->ctg_off[g]);
    for (uint64_t c = s->ctg_off[g]; c < s->ctg_off[g + 1]; c++) o.u32(s->ctg_len[c]);
  } else {
    o.u64(0);
  }
  o.u64(0);                                      // repetitive_kmers
  o.u64(d.nm);
  o.u64(s->sp.c); o.u64(s->sp.c); o.u64(s->sp.k);   // marker_c field = c (src/types.rs:347)
  o.u64(m->contig_order[i]);
  o.u8(0); o.u8(0);                              // individual_contig, amino_acid
}

// elements of blob array a in set s (ht_off is read for the table array only: a set growing in place extends it last)
uint64_t set_elems(const sk_sketch_set* s, int a) {
  const uint64_t n[N_COUNTS] = {s->S, s->U, s->M, s->C, SET_ARRAYS[a].by == CNT_HT ? s->ht_off[s->G] : 0};
  return array_elems(a, s->G, n);
}

// concatenate sketch sets (genome-local indexing everywhere, so only the prefix offsets shift).  with_tables: the parts
// carry their k-mer hash tables (ht_off / htab) and the result takes them over by copy instead of rebuilding them.
int concat_sets(sk_ctx* ctx, const std::vector<const sk_sketch_set*>& parts, sk_sketch_set** out, bool with_tables = false) {
  sk_sketch_set* s = new sk_sketch_set();
  s->ctx = ctx;
  s->sp = parts.empty() ? sk_sketch_params{125, 15, 1000} : parts[0]->sp;
  struct Guard { sk_sketch_set* s; ~Guard() { if (s) { free_set_device(s); delete s; } } } guard{s};
  s->seed_off = {0}; s->uk_off = {0}; s->mk_off = {0}; s->ctg_off = {0};
  if (with_tables) s->ht_off = {0};
  for (auto* p : parts) {
    if (!same_params(p->sp, s->sp)) { ctx->err = "sketch parameter mismatch"; return SK_ERR_PARAM; }
    for (uint32_t g = 0; g < p->G; g++) {
      s->seed_off.push_back(s->seed_off.back() + (p->seed_off[g + 1] - p->seed_off[g]));
      s->uk_off.push_back(s->uk_off.back() + (p->uk_off[g + 1] - p->uk_off[g]));
      s->mk_off.push_back(s->mk_off.back() + (p->mk_off[g + 1] - p->mk_off[g]));
      s->ctg_off.push_back(s->ctg_off.back() + (p->ctg_off[g + 1] - p->ctg_off[g]));
      if (with_tables) s->ht_off.push_back(s->ht_off.back() + (p->ht_off[g + 1] - p->ht_off[g]));
      s->total_len.push_back(p->total_len[g]);
      s->name_rank.push_back(s->G + g);
    }
    s->ctg_len.insert(s->ctg_len.end(), p->ctg_len.begin(), p->ctg_len.end());
    s->G += p->G;
  }
  s->S = s->seed_off.back(); s->U = s->uk_off.back(); s->M = s->mk_off.back(); s->C = s->ctg_off.back();
  for (int a = 0; a < BLOB_ARRAYS; a++) {
    if (!array_travels(a, false, with_tables)) continue;
    const size_t esz = SET_ARRAYS[a].esz;
    uint64_t total = 0;
    for (auto* p : parts) total += set_elems(p, a);
    SK_CUDA(ctx->arena.alloc(&set_array(s, a), std::max<uint64_t>(total, 1) * esz));
    uint8_t* dst = (uint8_t*)set_array(s, a);
    for (auto* p : parts) {
      const uint64_t n = set_elems(p, a);
      if (n) SK_CUDA(cudaMemcpyAsync(dst, set_array(p, a), n * esz, cudaMemcpyDeviceToDevice, ctx->stream));
      dst += n * esz;
    }
  }
  SK_CUDA(cudaStreamSynchronize(ctx->stream));
  guard.s = nullptr;
  *out = s;
  return SK_OK;
}

// The end of sk_sketch_set_import_batch and sk_sketch_set_import_blobs.  s (owned from here on: freed on failure) holds the
// host metadata: G, S, C, seed_off, ctg_off, ctg_len, total_len, name_rank.  rk / rp / rc hold the S records on the device,
// genome g's at seed_off[g] in any order; mraw the markers, genome g's at raw_off[g].  Range checks, each genome's records
// ordered by (contig, pos) ON THE DEVICE (one segmented radix sort over all genomes of the batch, so that a database of
// tens of thousands of sketches imports at PCIe speed; src/search.rs deserialises and re-hashes per pair), the per-contig
// first-record table with one sentinel per genome, then the views and hash tables.  rk / rp / rc are released before the
// views are built.
int import_finish(sk_ctx* ctx, sk_sketch_set* s, DTmp<uint32_t>& rk, DTmp<uint32_t>& rp, DTmp<uint32_t>& rc, DTmp<uint64_t>& mraw,
                  const std::vector<uint64_t>& raw_off, sk_sketch_set** out) {
  struct Guard { sk_sketch_set* s; ~Guard() { if (s) { free_set_device(s); delete s; } } } guard{s};
  const uint32_t G = s->G;
  const uint64_t n_records = s->S, n_contigs = s->C, n_markers = raw_off[G];
  const sk_sketch_params* sp = &s->sp;
  const size_t S1 = std::max<size_t>(n_records, 1);
  SK_CUDA(ctx->arena.alloc((void**)&s->pv_kmer, S1 * 4)); SK_CUDA(ctx->arena.alloc((void**)&s->pv_pos, S1 * 4));
  SK_CUDA(ctx->arena.alloc((void**)&s->pv_cc, S1 * 4));
  SK_CUDA(ctx->arena.alloc((void**)&s->d_ctg_len, std::max<size_t>(n_contigs, 1) * 4));
  SK_CUDA(ctx->arena.alloc((void**)&s->ctg_rec_off, (size_t)(n_contigs + G + 1) * 4));
  cudaStream_t st = ctx->stream;
  SK_CUDA(cudaStreamSynchronize(st));
  if (n_contigs) SK_CUDA(cudaMemcpyAsync(s->d_ctg_len, s->ctg_len.data(), n_contigs * 4, cudaMemcpyHostToDevice, st));
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
    if (n_markers) {
      import_range_kernel<uint64_t><<<range_blocks(n_markers), 256, 0, st>>>(mraw.p, n_markers, 1ull << (2 * MARKER_K), d_bad.p, BAD_MARKER);
      count_launch(ctx);
    }
    if (n_records) {
      DTmp<uint32_t> vals, perm;
      DTmp<uint64_t> keys, skeys;
      SK_CUDA(vals.alloc(n_records, ctx)); SK_CUDA(perm.alloc(n_records, ctx)); SK_CUDA(keys.alloc(n_records, ctx)); SK_CUDA(skeys.alloc(n_records, ctx));
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
    rk.release(); rp.release(); rc.release();
    uint32_t bad = 0;
    SK_CUDA(cudaMemcpyAsync(&bad, d_bad.p, 4, cudaMemcpyDeviceToHost, st));
    SK_CUDA(cudaStreamSynchronize(st));
    if (bad & BAD_MARKER) { ctx->err = "marker out of range (markers must be < 2^42)"; return SK_ERR_PARAM; }
    if (bad & BAD_KMER) { ctx->err = "seed k-mer out of range (k-mers must be < 4^k)"; return SK_ERR_PARAM; }
    if (bad & BAD_CONTIG) { ctx->err = "record contig index out of range"; return SK_ERR_PARAM; }
  }
  mbox_reset(ctx);                 // build_views takes pinned read-back space from the context's mailbox
  SK_TRY(build_views(ctx, s, mraw.p, raw_off.data()));
  SK_TRY(build_hash(ctx, s));
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

int sk_sketch_set_blob_size(const sk_sketch_set* s, uint64_t* device_bytes, uint64_t* host_meta_words) {
  return sk_sketch_set_subset_blob_size(s, nullptr, 0, 0, device_bytes, host_meta_words);
}

int sk_sketch_set_pack(const sk_sketch_set* s, void* d_blob, uint64_t* meta) { return sk_sketch_set_pack_subset(s, nullptr, 0, 0, d_blob, meta); }

namespace {
// metadata of a subset blob: the selected genomes (genomes = NULL: all) in output order
int plan_subset(const sk_sketch_set* s, const uint32_t* genomes, uint32_t n, int flags, std::vector<uint32_t>& idx, SetMeta& m) {
  const bool mo = (flags & SK_PACK_MARKERS_ONLY) != 0;
  if (!genomes) { n = s->G; idx.resize(n); for (uint32_t i = 0; i < n; i++) idx[i] = i; }
  else idx.assign(genomes, genomes + n);
  m.c = s->sp.c; m.k = s->sp.k; m.marker_c = s->sp.marker_c;
  m.tables = !mo && (flags & SK_PACK_TABLES) != 0 && s->htab != nullptr && s->ht_off.size() == (size_t)s->G + 1;
  for (uint32_t g : idx) {
    if (g >= s->G) { s->ctx->err = "subset genome index out of range"; return SK_ERR_PARAM; }
    const uint64_t cnt[N_COUNTS] = {s->seed_off[g + 1] - s->seed_off[g], s->uk_off[g + 1] - s->uk_off[g], s->mk_off[g + 1] - s->mk_off[g],
                                    s->ctg_off[g + 1] - s->ctg_off[g], m.tables ? s->ht_off[g + 1] - s->ht_off[g] : 0};
    meta_push(m, cnt, mo, s->total_len[g], s->ctg_len.begin() + s->ctg_off[g], s->ctg_len.begin() + s->ctg_off[g + 1]);
  }
  return SK_OK;
}
}  // namespace

int sk_sketch_set_subset_blob_size(const sk_sketch_set* s, const uint32_t* genomes, uint32_t n, int flags, uint64_t* device_bytes,
                                   uint64_t* host_meta_words) {
  if (!s || !device_bytes || !host_meta_words) return SK_ERR_PARAM;
  std::vector<uint32_t> idx;
  SetMeta m;
  SK_TRY(plan_subset(s, genomes, n, flags, idx, m));
  *device_bytes = blob_layout(m.G, m.n).total;
  *host_meta_words = meta_words(m.G, m.n[CNT_C], m.tables);
  return SK_OK;
}

int sk_sketch_set_pack_subset(const sk_sketch_set* s, const uint32_t* genomes, uint32_t n, int flags, void* d_blob, uint64_t* meta) {
  if (!s || !d_blob || !meta) return SK_ERR_PARAM;
  sk_ctx* ctx = s->ctx;
  SK_CUDA(cudaSetDevice(ctx->device));
  std::vector<uint32_t> idx;
  SetMeta m;
  SK_TRY(plan_subset(s, genomes, n, flags, idx, m));
  const bool mo = (flags & SK_PACK_MARKERS_ONLY) != 0;
  const uint32_t G = (uint32_t)m.G;
  const BlobLayout b = blob_layout(G, m.n);
  uint8_t* base = (uint8_t*)d_blob;
  SK_CUDA(zero_absent_arrays(ctx, base, b, mo, m.tables));
  // maximal runs of consecutive source genomes [a, e) -> one segment per array; a scattered subset (the cross-block fetch of a
  // genome order unrelated to relatedness asks for thousands of runs: 150 ms measured for 5 000 genomes as separate calls)
  // goes through the batched copy beyond a few runs
  const std::vector<uint64_t>* src[N_COUNTS] = {&s->seed_off, &s->uk_off, &s->mk_off, &s->ctg_off, &s->ht_off};
  std::vector<std::pair<uint32_t, uint32_t>> runs;   // [i, j) of the output
  for (uint32_t i = 0; i < G;) {
    uint32_t j = i + 1;
    while (j < G && idx[j] == idx[j - 1] + 1) j++;
    runs.push_back({i, j});
    i = j;
  }
  SegmentCopy cp;
  cp.batched = runs.size() > 8;
  for (auto [i, j] : runs) {
    const uint32_t a0 = idx[i], e = idx[j - 1] + 1;
    for (int a = 0; a < BLOB_ARRAYS; a++) {
      if (!array_travels(a, mo, m.tables)) continue;
      const ArrayDesc& d = SET_ARRAYS[a];
      const std::vector<uint64_t>& so = *src[d.by];
      const uint64_t first = array_index(a, a0, so[a0]), count = array_index(a, e, so[e]) - first;
      cp.add((const uint8_t*)set_array(s, a) + first * d.esz, base + b.off[a] + array_index(a, i, m.off[d.by][i]) * d.esz, count * d.esz);
    }
  }
  SK_TRY(cp.run(ctx));
  encode_meta(m, meta);
  SK_CUDA(cudaStreamSynchronize(ctx->stream));
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
    SetMeta m = decode_meta(metas[i]);
    sk_sketch_set& v = views[i];
    v.ctx = ctx;
    v.G = (uint32_t)m.G; v.S = m.n[CNT_S]; v.U = m.n[CNT_U]; v.M = m.n[CNT_M]; v.C = m.n[CNT_C];
    v.sp = sk_sketch_params{(uint32_t)m.c, (uint32_t)m.k, (uint32_t)m.marker_c};
    all_tables = all_tables && (m.tables || v.U == 0);
    v.seed_off = std::move(m.off[CNT_S]); v.uk_off = std::move(m.off[CNT_U]); v.mk_off = std::move(m.off[CNT_M]);
    v.ctg_off = std::move(m.off[CNT_C]); v.ht_off = std::move(m.off[CNT_HT]);
    v.total_len = std::move(m.total_len);
    v.ctg_len.assign(m.ctg_len.begin(), m.ctg_len.end());
    v.name_rank.resize(v.G);
    const BlobLayout b = blob_layout(m.G, m.n);
    for (int a = 0; a < BLOB_ARRAYS; a++) set_array(&v, a) = (uint8_t*)d_blobs[i] + b.off[a];
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
  const bool pinned_src = prepacked ? (host_pinned(seq.units) && (!seq.nmask || host_pinned(seq.nmask))) : host_pinned(seq.ascii);
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
// appends `add` elements of esz bytes at element `used` of *arr, growing it by 1.5x when its capacity (0: exactly `used`) is short
int grow_append(sk_ctx* ctx, void*& arr, size_t& cap, size_t used, const void* src, size_t add, size_t esz) {
  const size_t have = cap ? cap : std::max<size_t>(used, 1);
  if (used + add > have) {
    const size_t ncap = std::max<size_t>(used + add, have + have / 2);
    void* n = nullptr;
    SK_CUDA(ctx->arena.alloc(&n, ncap * esz));
    if (used) SK_CUDA(cudaMemcpyAsync(n, arr, used * esz, cudaMemcpyDeviceToDevice, ctx->stream));
    SK_CUDA(cudaStreamSynchronize(ctx->stream));
    if (arr) ctx->arena.release(arr);
    arr = n; cap = ncap;
  }
  if (add) SK_CUDA(cudaMemcpyAsync((uint8_t*)arr + used * esz, src, add * esz, cudaMemcpyDeviceToDevice, ctx->stream));
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
    // distinct k-mers <= records; table capacity = power of two >= 2 x distinct k-mers: between 2 and 4 entries per k-mer.
    // Sized for one genome and one contig more than the hint, so ctg_rec_off (contig + genome counted) holds one element more
    // than the hint can need
    const uint64_t reserve[N_COUNTS] = {S, S, M, hint.contigs + 1, 4 * S + 16 * hint.genomes};
    struct G0 { sk_sketch_set* s; ~G0() { if (s) { free_set_device(s); delete s; } } } g0{d};
    for (int a = 0; a < BLOB_ARRAYS; a++) {
      d->cap[a] = array_elems(a, hint.genomes + 1, reserve);
      SK_CUDA(ctx->arena.alloc(&set_array(d, a), d->cap[a] * SET_ARRAYS[a].esz));
    }
    g0.s = nullptr;
    *dstp = d;
  }
  const uint32_t g_begin = d->G;
  for (auto* p : parts) {
    if (!same_params(p->sp, d->sp)) { ctx->err = "sketch parameter mismatch"; return SK_ERR_PARAM; }
    for (int a = 0; a < BLOB_ARRAYS; a++)   // every array but the k-mer tables, which build_hash_range appends
      if (array_travels(a, false, false))
        SK_TRY(grow_append(ctx, set_array(d, a), d->cap[a], set_elems(d, a), set_array(p, a), set_elems(p, a), SET_ARRAYS[a].esz));
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
  std::vector<uint64_t> raw_off(G + 1);
  for (uint32_t g = 0; g <= G; g++) raw_off[g] = mk_off[g] - m0;
  cudaStream_t st = ctx->stream;
  DTmp<uint64_t> mraw;
  DTmp<uint32_t> rk, rp, rc;
  SK_CUDA(mraw.alloc(n_markers, ctx));
  if (n_markers) SK_CUDA(cudaMemcpyAsync(mraw.p, markers + m0, n_markers * 8, cudaMemcpyHostToDevice, st));
  if (n_records) {
    SK_CUDA(rk.alloc(n_records, ctx)); SK_CUDA(rp.alloc(n_records, ctx)); SK_CUDA(rc.alloc(n_records, ctx));
    SK_CUDA(cudaMemcpyAsync(rk.p, kmer + r0, n_records * 4, cudaMemcpyHostToDevice, st));
    SK_CUDA(cudaMemcpyAsync(rp.p, pos + r0, n_records * 4, cudaMemcpyHostToDevice, st));
    SK_CUDA(cudaMemcpyAsync(rc.p, cc + r0, n_records * 4, cudaMemcpyHostToDevice, st));
  }
  guard.s = nullptr;
  return import_finish(ctx, s, rk, rp, rc, mraw, raw_off, out);
}

int sk_sketch_set_import_blobs(sk_ctx* ctx, const sk_sketch_params* sp, const uint8_t* bytes, const uint64_t* blob_off,
                               const uint64_t* blob_len, uint32_t n_blobs, sk_sketch_set** out, uint32_t* bad_blob) {
  if (bad_blob) *bad_blob = UINT32_MAX;
  if (!ctx || !out || n_blobs == 0 || !bytes || !blob_off || !blob_len) return SK_ERR_PARAM;
  SK_CUDA(cudaSetDevice(ctx->device));
  SK_TRY(check_sketch_params(ctx, sp));
  const uint32_t G = n_blobs;
  auto refuse = [&](uint32_t g, const std::string& why) {
    ctx->err = "sketch blob " + std::to_string(g) + ": " + why;
    if (bad_blob) *bad_blob = g;
    return SK_ERR_PARAM;
  };
  // ---- host: the framing of every blob (skdb::scan_entry), on the worker pool
  std::vector<skdb::SketchScan> sc(G);
  std::vector<std::string> why(G);
  ctx_pool(ctx)->run(G, [&](size_t g) {
    try {
      sc[g] = skdb::scan_entry(bytes + blob_off[g], blob_len[g]);
      const skdb::DiskParams& p = sc[g].params;
      if (p.use_aa) why[g] = "amino-acid sketches are not supported";
      else if (p.c != sp->c || p.k != sp->k || p.marker_c != sp->marker_c) why[g] = "sketch parameters differ from the call's";
    } catch (const std::exception& e) { why[g] = e.what(); }
  });
  for (uint32_t g = 0; g < G; g++) if (!why[g].empty()) return refuse(g, why[g]);
  // ---- descriptors (blob g's bytes land at dev_at in the device copy, the blobs back to back) and host metadata
  sk_sketch_set* s = new sk_sketch_set();
  s->ctx = ctx; s->sp = *sp; s->G = G;
  struct Guard { sk_sketch_set* s; ~Guard() { if (s) { free_set_device(s); delete s; } } } guard{s};
  std::vector<BlobDesc> desc(G);
  std::vector<uint64_t> list_at, list_len, raw_off(G + 1, 0);
  std::vector<std::pair<const uint8_t*, uint64_t>> runs;
  s->ctg_off.assign(1, 0);
  uint64_t K = 0, M = 0, dev_at = 0;
  for (uint32_t g = 0; g < G; g++) {
    const skdb::SketchScan& x = sc[g];
    const uint8_t* p = bytes + blob_off[g];
    desc[g] = BlobDesc{dev_at + x.keys_at, K, x.n_keys, list_at.size(), x.multi_at.size(), dev_at + x.markers_at, M, x.n_markers};
    for (size_t j = 0; j < x.multi_at.size(); j++) { list_at.push_back(dev_at + x.multi_at[j]); list_len.push_back(x.multi_len[j]); }
    for (uint64_t c = 0; c < x.n_ctg_len; c++) s->ctg_len.push_back(skdb::load_u32(p + x.ctg_len_at + 4 * c));
    s->ctg_off.push_back(s->ctg_len.size());
    s->total_len.push_back(x.total_len);
    s->name_rank.push_back(g);
    K += x.n_keys; M += x.n_markers;
    raw_off[g + 1] = M;
    if (!runs.empty() && runs.back().first + runs.back().second == p) runs.back().second += blob_len[g];   // adjacent in memory
    else runs.push_back({p, blob_len[g]});
    dev_at += blob_len[g];
  }
  s->C = s->ctg_len.size();
  if (K + 1 >= (1ull << 31) || M >= (1ull << 31) || s->C >= (1ull << 31)) {
    ctx->err = "import batch too large (>= 2^31 keys, markers or contigs): import in several batches and sk_sketch_set_append";
    return SK_ERR_PARAM;
  }
  // ---- device: the bytes as stored, the count of every key's records, their exclusive scan, then the expansion.  The
  //      bytes are released before import_finish takes its sort temporaries: the peak stays below sk_sketch_set_import_batch's
  //      for the same records (bytes ~ 12 per record + 8 per marker, against 32 per record of sort temporaries there)
  cudaStream_t st = ctx->stream;
  DTmp<uint8_t> dbuf;
  DTmp<BlobDesc> d_desc;
  DTmp<uint64_t> d_list_at, d_list_len, key_rec, d_ro;
  DTmp<uint32_t> d_bad;
  SK_CUDA(dbuf.alloc(dev_at + 16, ctx));
  SK_CUDA(d_desc.alloc(G, ctx)); SK_CUDA(d_list_at.alloc(list_at.size(), ctx)); SK_CUDA(d_list_len.alloc(list_len.size(), ctx));
  SK_CUDA(key_rec.alloc(K + 1, ctx)); SK_CUDA(d_ro.alloc(G + 1, ctx)); SK_CUDA(d_bad.alloc(1, ctx));
  SK_CUDA(cudaMemsetAsync(dbuf.p + dev_at, 0, 16, st));
  SK_TRY(upload_runs(ctx, dbuf.p, runs, host_pinned(bytes)));
  SK_CUDA(cudaMemcpyAsync(d_desc.p, desc.data(), G * sizeof(BlobDesc), cudaMemcpyHostToDevice, st));
  if (!list_at.empty()) {
    SK_CUDA(cudaMemcpyAsync(d_list_at.p, list_at.data(), list_at.size() * 8, cudaMemcpyHostToDevice, st));
    SK_CUDA(cudaMemcpyAsync(d_list_len.p, list_len.data(), list_len.size() * 8, cudaMemcpyHostToDevice, st));
  }
  SK_CUDA(cudaMemsetAsync(d_bad.p, 0xFF, 4, st));
  SK_CUDA(cudaMemsetAsync(key_rec.p + K, 0, 8, st));
  if (K) { blob_count_kernel<<<dim3(G, 8), 256, 0, st>>>(dbuf.p, d_desc.p, d_list_len.p, key_rec.p, d_bad.p); count_launch(ctx); }
  {
    size_t tb = 0;
    SK_CUDA(cub::DeviceScan::ExclusiveSum(nullptr, tb, key_rec.p, key_rec.p, (int)(K + 1), st));
    DTmp<uint8_t> tmp;
    SK_CUDA(tmp.alloc(tb, ctx));
    SK_CUDA(cub::DeviceScan::ExclusiveSum(tmp.p, tb, key_rec.p, key_rec.p, (int)(K + 1), st));
    count_launch(ctx);
  }
  blob_rec_off_kernel<<<(G + 256) / 256, 256, 0, st>>>(d_desc.p, G, K, key_rec.p, d_ro.p); count_launch(ctx);
  s->seed_off.resize(G + 1);
  uint32_t bad = UINT32_MAX;
  SK_CUDA(cudaMemcpyAsync(s->seed_off.data(), d_ro.p, (G + 1) * 8, cudaMemcpyDeviceToHost, st));
  SK_CUDA(cudaMemcpyAsync(&bad, d_bad.p, 4, cudaMemcpyDeviceToHost, st));
  SK_CUDA(cudaStreamSynchronize(st));
  if (bad != UINT32_MAX) return refuse(bad, "multi-position index out of range");
  s->S = s->seed_off[G];
  if (s->S >= (1ull << 31)) { ctx->err = "import batch too large (>= 2^31 records): import in several batches and sk_sketch_set_append"; return SK_ERR_PARAM; }
  DTmp<uint32_t> rk, rp, rc;
  DTmp<uint64_t> mraw;
  SK_CUDA(rk.alloc(s->S, ctx)); SK_CUDA(rp.alloc(s->S, ctx)); SK_CUDA(rc.alloc(s->S, ctx)); SK_CUDA(mraw.alloc(M, ctx));
  if (s->S) {
    blob_expand_kernel<<<dim3(G, 8), 256, 0, st>>>(dbuf.p, d_desc.p, d_list_at.p, d_list_len.p, key_rec.p, rk.p, rp.p, rc.p);
    count_launch(ctx);
  }
  if (M) { blob_markers_kernel<<<dim3(G, 8), 256, 0, st>>>(dbuf.p, d_desc.p, mraw.p); count_launch(ctx); }
  SK_CUDA(cudaGetLastError());
  dbuf.release(); key_rec.release(); d_list_at.release(); d_list_len.release(); d_desc.release();
  guard.s = nullptr;
  return import_finish(ctx, s, rk, rp, rc, mraw, raw_off, out);
}

int sk_sketch_set_import(sk_ctx* ctx, const sk_sketch_params* sp, const uint32_t* kmer, const uint32_t* pos,
                         const uint32_t* cc, uint64_t n_records, const uint64_t* markers, uint64_t n_markers,
                         const uint32_t* contig_lengths, uint32_t n_contigs, sk_sketch_set** out) {
  const uint64_t ro[2] = {0, n_records}, mo[2] = {0, n_markers}, co[2] = {0, n_contigs};
  return sk_sketch_set_import_batch(ctx, sp, 1, ro, kmer, pos, cc, mo, markers, co, contig_lengths, nullptr, out);
}

int sk_sketch_set_encode_sizes(const sk_sketch_set* s, uint32_t g0, uint32_t n, int form, const sk_entry_meta* meta, uint64_t* entry_len) {
  if (!s) return SK_ERR_PARAM;
  sk_ctx* ctx = s->ctx;
  SK_TRY(check_encode_args(ctx, s, g0, n, form, meta));
  if (n == 0) return SK_OK;
  if (!entry_len) { ctx->err = "encode: entry_len is required"; return SK_ERR_PARAM; }
  SK_CUDA(cudaSetDevice(ctx->device));
  EncodeJob j{s, g0, n, form == SK_ENTRY_FULL, meta, {}, {}};
  encode_job_init(j);
  DTmp<EncDesc> d_desc;
  DTmp<uint32_t> scan;
  if (j.full) SK_TRY(count_multi(ctx, j, d_desc, scan));
  encode_layout(j);
  for (uint32_t i = 0; i < n; i++) entry_len[i] = j.lay[i].length;
  return SK_OK;
}

int sk_sketch_set_encode(const sk_sketch_set* s, uint32_t g0, uint32_t n, int form, const sk_entry_meta* meta, uint8_t* out, uint64_t out_cap,
                         uint64_t* entry_len) {
  if (!s) return SK_ERR_PARAM;
  sk_ctx* ctx = s->ctx;
  SK_TRY(check_encode_args(ctx, s, g0, n, form, meta));
  if (n == 0) return SK_OK;
  SK_CUDA(cudaSetDevice(ctx->device));
  cudaStream_t st = ctx->stream;
  EncodeJob j{s, g0, n, form == SK_ENTRY_FULL, meta, {}, {}};
  encode_job_init(j);
  DTmp<EncDesc> d_all;
  DTmp<uint32_t> scan;
  if (j.full) SK_TRY(count_multi(ctx, j, d_all, scan));
  const uint64_t total = encode_layout(j);
  if (!out || out_cap < total) { ctx->err = "encode: the output buffer holds " + std::to_string(out_cap) + " bytes, the entries take " + std::to_string(total); return SK_ERR_PARAM; }
  if (entry_len) for (uint32_t i = 0; i < n; i++) entry_len[i] = j.lay[i].length;
  const bool pinned = host_pinned(out);
  // entries in chunks of about CHUNK bytes (at least one entry), each written into one device buffer and copied out
  const uint64_t CHUNK = 1ull << 30;
  for (uint32_t a = 0; a < n;) {
    uint32_t b = a + 1;
    while (b < n && j.desc[b].at + j.lay[b].length - j.desc[a].at <= CHUNK) b++;
    const uint64_t base = j.desc[a].at, bytes = j.desc[b - 1].at + j.lay[b - 1].length - base;
    std::vector<EncDesc> cd(j.desc.begin() + a, j.desc.begin() + b);
    skdb::Out host;
    for (uint32_t i = a; i < b; i++) {
      EncDesc& d = cd[i - a];
      d.at -= base; d.keys_at -= base; d.multi_at -= base; d.markers_at -= base; d.mid_at -= base; d.tail_at -= base;
      d.host_at = host.b.size();
      encode_host_sections(j, i, host);
      if (host.b.size() - d.host_at != d.head_len + d.mid_len + d.tail_len) { ctx->err = "encode: host sections disagree with the entry layout"; return SK_ERR_STATE; }
    }
    DTmp<uint8_t> dbuf, dhost;
    DTmp<EncDesc> d_desc;
    SK_CUDA(dbuf.alloc(bytes, ctx)); SK_CUDA(dhost.alloc(host.b.size(), ctx)); SK_CUDA(d_desc.alloc(b - a, ctx));
    SK_CUDA(cudaMemcpyAsync(d_desc.p, cd.data(), cd.size() * sizeof(EncDesc), cudaMemcpyHostToDevice, st));
    SK_CUDA(cudaMemcpyAsync(dhost.p, host.b.data(), host.b.size(), cudaMemcpyHostToDevice, st));
    enc_write_kernel<<<dim3(b - a, 8), 256, 0, st>>>(d_desc.p, s->ukmer, s->ustart, s->kv_pos, s->kv_cc, s->markers, j.full ? scan.p : nullptr,
                                                     dhost.p, dbuf.p);
    count_launch(ctx);
    SK_CUDA(cudaGetLastError());
    SK_TRY(download_bytes(ctx, out + base, dbuf.p, bytes, pinned));
    a = b;
  }
  return SK_OK;
}

}  // extern "C"
