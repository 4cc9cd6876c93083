// screen.cu -- marker prefilter on the device.
//
// Replaces screen::kmer_to_sketch_from_refs (reference src/screen.rs:190-210, a serial hash-map build) and
// screen_refs / screen_refs_indices / check_markers_quickly (src/screen.rs:148, 39, 84).
//
// The inverted index marker -> [sketch ids] becomes one radix sort of all (marker, entry) pairs: equal markers
// form a run, and because the sort is stable and entries are laid out genome-major, the members of a run are in
// ascending genome order.  A row (query genome) then counts shared markers per column genome in shared memory by
// walking, for each of its markers, the slice of the run that holds the column entries:
//   triangle   : columns = entries after its own position in the run (only j > i is ever used, src/triangle.rs:90)
//   query x ref: ref entries precede query entries inside a run (refs are laid out first)
// and applies the exact integer/f64 predicate of the reference to every column.
#include <cub/cub.cuh>

#include <algorithm>
#include <cstdlib>
#include <cstring>

#include "sk_core.cuh"
#include "sk_internal.h"

namespace sk {

static inline uint32_t div_up64(uint64_t a, uint32_t b) { return (uint32_t)((a + b - 1) / b); }

// f64::powi(x, 21) as compiler-rt's __powidf2 / LLVM's powi expansion evaluate it (square-and-multiply from the
// low bit); reference src/screen.rs:60,124,176
static double powi21(double x) {
  double r = 1.0, a = x;
  int b = MARKER_K;
  while (true) {
    if (b & 1) r *= a;
    b /= 2;
    if (b == 0) break;
    a *= a;
  }
  return r;
}

double screen_cutoff(const sk_map_params* mp) { return powi21(mp->screen_val == 0. ? 0.80 : mp->screen_val); }   // src/triangle.rs:34-42

__global__ void fill_genome_kernel(const uint64_t* __restrict__ off, uint32_t base_entry, uint32_t* __restrict__ eg) {
  uint32_t g = blockIdx.x;
  for (uint64_t i = off[g] + threadIdx.x; i < off[g + 1]; i += blockDim.x) eg[base_entry + i] = g;
}
__global__ void iota_kernel(uint32_t* v, uint32_t n) {
  uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) v[i] = i;
}
__global__ void run_head_kernel(const uint64_t* __restrict__ key, uint32_t n, uint32_t* __restrict__ head) {
  uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) head[i] = (i == 0 || key[i] != key[i - 1]) ? 1u : 0u;
}
// rstart[run] = first sorted position of the run; rstart[n_runs] = n
__global__ void run_start_kernel(const uint32_t* __restrict__ head, const uint32_t* __restrict__ hscan, uint32_t n,
                                 uint32_t n_runs, uint32_t* __restrict__ rstart) {
  uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n && head[i]) rstart[hscan[i]] = i;
  if (i == 0) rstart[n_runs] = n;
}
// triangle: entry e at sorted position p sees the rest of its run
__global__ void tri_ranges_kernel(const uint32_t* __restrict__ sval, const uint32_t* __restrict__ head,
                                  const uint32_t* __restrict__ hscan, const uint32_t* __restrict__ rstart,
                                  const uint32_t* __restrict__ eg, uint32_t n, uint32_t* __restrict__ ra,
                                  uint32_t* __restrict__ rb, uint32_t* __restrict__ scol) {
  uint32_t p = blockIdx.x * blockDim.x + threadIdx.x;
  if (p >= n) return;
  uint32_t e = sval[p];
  uint32_t run = hscan[p] + head[p] - 1;
  ra[e] = p + 1;
  rb[e] = rstart[run + 1];
  scol[p] = eg[e];
}
// query x ref: refs are entries [0, n_ref); inside a run they precede the query entries
__global__ void qr_firstq_kernel(const uint32_t* __restrict__ sval, const uint32_t* __restrict__ head,
                                 const uint32_t* __restrict__ hscan, uint32_t n, uint32_t n_ref,
                                 uint32_t* __restrict__ firstq) {
  uint32_t p = blockIdx.x * blockDim.x + threadIdx.x;
  if (p >= n) return;
  if (sval[p] >= n_ref && (head[p] || sval[p - 1] < n_ref)) firstq[hscan[p] + head[p] - 1] = p;
}
__global__ void qr_ranges_kernel(const uint32_t* __restrict__ sval, const uint32_t* __restrict__ head,
                                 const uint32_t* __restrict__ hscan, const uint32_t* __restrict__ rstart,
                                 const uint32_t* __restrict__ firstq, const uint32_t* __restrict__ eg, uint32_t n,
                                 uint32_t n_ref, uint32_t* __restrict__ ra, uint32_t* __restrict__ rb,
                                 uint32_t* __restrict__ scol) {
  uint32_t p = blockIdx.x * blockDim.x + threadIdx.x;
  if (p >= n) return;
  uint32_t e = sval[p];
  uint32_t run = hscan[p] + head[p] - 1;
  if (e >= n_ref) {
    ra[e - n_ref] = rstart[run];
    rb[e - n_ref] = firstq[run];
    scol[p] = 0xFFFFFFFFu;
  } else {
    scol[p] = eg[e];
  }
}

// One block per row genome.  counts[] lives in dynamic shared memory (tile of `tile` columns).
__global__ void __launch_bounds__(256)
screen_rows_kernel(const uint64_t* __restrict__ row_mk_off, const uint64_t* __restrict__ col_mk_off, uint32_t n_rows,
                   uint32_t n_cols, const uint32_t* __restrict__ ra, const uint32_t* __restrict__ rb,
                   const uint32_t* __restrict__ scol, int mode, int rescue_small, double cutoff, int all_pass,
                   uint32_t tile, uint64_t* __restrict__ pairs, unsigned long long* __restrict__ n_pairs,
                   unsigned long long cap, uint32_t row_mod, uint32_t row_rem) {
  extern __shared__ uint32_t counts[];
  const uint32_t i = blockIdx.x * row_mod + row_rem;
  if (i >= n_rows) return;
  const uint64_t mb = row_mk_off[i], me = row_mk_off[i + 1];
  const uint64_t card_i = me - mb;
  const bool tri = (mode == MODE_TRIANGLE);
  const uint32_t col_begin = tri ? i + 1 : 0;
  // a rescued row passes every column: nothing to count
  const bool row_rescue = screen_row_rescued(mode, rescue_small, card_i);
  for (uint32_t t0 = col_begin; t0 < n_cols; t0 += tile) {
    const uint32_t t1 = min(n_cols, t0 + tile);
    for (uint32_t c = threadIdx.x; c < t1 - t0; c += blockDim.x) counts[c] = 0;
    __syncthreads();
    if (!row_rescue && !all_pass) {
      for (uint64_t e = mb + threadIdx.x; e < me; e += blockDim.x) {
        uint32_t a = ra[e], b = rb[e];
        for (uint32_t t = a; t < b; t++) {
          uint32_t col = scol[t];
          if (col >= t0 && col < t1) atomicAdd(&counts[col - t0], 1u);
        }
      }
    }
    __syncthreads();
    for (uint32_t c = threadIdx.x; c < t1 - t0; c += blockDim.x) {
      const uint32_t j = t0 + c;
      const uint64_t card_j = col_mk_off[j + 1] - col_mk_off[j];
      if (all_pass || screen_pass(mode, rescue_small, card_i, card_j, counts[c], cutoff)) {
        unsigned long long slot = atomicAdd(n_pairs, 1ull);
        // triangle: (i, j); query x ref: (ref = column, query = row)
        if (slot < cap) pairs[slot] = tri ? (((uint64_t)i << 32) | j) : (((uint64_t)j << 32) | i);
      }
    }
    __syncthreads();
  }
}

// The row pass of a screen whose ra / rb / scol are laid out: screen_rows_kernel over the rows (row_mod, row_rem) of
// [0, n_rows_total) against the columns [0, NC) (col_off[j] .. col_off[j + 1] = column j's markers), with a first pair buffer of
// max(2^20, 64 * cap_rows) pairs and one retry at the exact count when it overflows; the pairs are sorted and returned in a
// malloc'd host array.
static int rows_pass(sk_ctx* ctx, const uint64_t* d_row_off, const uint64_t* d_col_off, uint32_t n_rows_total, uint32_t NC,
                     const uint32_t* ra, const uint32_t* rb, const uint32_t* scol, int mode, int rescue_small, double cutoff,
                     uint32_t cap_rows, uint32_t row_mod, uint32_t row_rem, uint64_t** out_pairs, uint64_t* out_n) {
  cudaStream_t st = ctx->stream;
  // check_markers_quickly returns true outright for screen_val == 0 (src/screen.rs:91-93); callers substitute the default
  // first, so this only triggers for an explicit 0 that survived: never through the reference CLI.
  const int all_pass = 0;
  const uint32_t tile = std::min<uint32_t>(NC, 48 * 1024);
  const size_t smem = (size_t)tile * 4;
  // always the same (maximal) value: the attribute is per device, and several contexts may screen on one device concurrently
  SK_CUDA(cudaFuncSetAttribute(screen_rows_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 48 * 1024 * 4));
  unsigned long long cap = std::max<unsigned long long>(1ull << 20, 64ull * cap_rows);
  DTmp<unsigned long long> d_n;
  SK_CUDA(d_n.alloc(1, ctx));
  DTmp<uint64_t> d_pairs;
  unsigned long long n = 0;
  for (int attempt = 0; attempt < 2; attempt++) {
    SK_CUDA(d_pairs.alloc(cap, ctx));
    SK_CUDA(cudaMemsetAsync(d_n.p, 0, 8, st));
    const uint32_t n_rows_launch = n_rows_total > row_rem ? (n_rows_total - row_rem + row_mod - 1) / row_mod : 0;
    if (n_rows_launch) {
      SK_LAUNCH(ctx, "screen_rows_kernel", (screen_rows_kernel<<<n_rows_launch, 256, smem, st>>>(
          d_row_off, d_col_off, n_rows_total, NC, ra, rb, scol, mode, rescue_small, cutoff, all_pass, tile, d_pairs.p, d_n.p, cap,
          row_mod, row_rem)));
    }
    SK_CUDA(cudaMemcpyAsync(&n, d_n.p, 8, cudaMemcpyDeviceToHost, st));
    SK_CUDA(cudaStreamSynchronize(st));
    SK_CUDA(cudaGetLastError());
    if (n <= cap) break;
    cap = n;
  }
  uint64_t* host = (uint64_t*)malloc(std::max<size_t>(n, 1) * 8);
  if (!host) return SK_ERR_NOMEM;
  if (n > 0) {
    DTmp<uint64_t> sorted;
    SK_CUDA(sorted.alloc(n, ctx));
    size_t tb = 0;
    SK_CUDA(cub::DeviceRadixSort::SortKeys(nullptr, tb, d_pairs.p, sorted.p, (uint64_t)n, 0, 64, st));
    DTmp<uint8_t> tmp;
    SK_CUDA(tmp.alloc(tb, ctx));
    SK_CUDA(cub::DeviceRadixSort::SortKeys(tmp.p, tb, d_pairs.p, sorted.p, (uint64_t)n, 0, 64, st));
    SK_CUDA(cudaMemcpyAsync(host, sorted.p, n * 8, cudaMemcpyDeviceToHost, st));
    SK_CUDA(cudaStreamSynchronize(st));
  }
  *out_pairs = host;
  *out_n = n;
  return SK_OK;
}

static int run_screen(sk_ctx* ctx, const sk_sketch_set* rows, const sk_sketch_set* cols, int mode, const sk_map_params* mp,
                      uint64_t** out_pairs, uint64_t* out_n, uint32_t row_mod = 1, uint32_t row_rem = 0) {
  cudaStream_t st = ctx->stream;
  const bool tri = (mode == MODE_TRIANGLE);
  const uint32_t NR = rows->G, NC = cols->G;
  *out_pairs = nullptr; *out_n = 0;
  if (NR == 0 || NC == 0) { *out_pairs = (uint64_t*)malloc(8); return SK_OK; }
  const size_t Mc = cols->M, Mr = tri ? 0 : rows->M;
  const size_t N = Mc + Mr;  // sorted entries: column (ref) entries first, then row (query) entries
  if (N >= (1ull << 31)) { ctx->err = "marker table too large for one screen call (>= 2^31 entries)"; return SK_ERR_PARAM; }
  double screen_val = mp->screen_val == 0. ? 0.80 : mp->screen_val;  // src/triangle.rs:34-42, src/dist.rs:68-77
  const double cutoff = powi21(screen_val);

  DTmp<uint64_t> d_row_off, d_col_off;
  SK_CUDA(d_row_off.alloc(NR + 1, ctx)); SK_CUDA(d_col_off.alloc(NC + 1, ctx));
  SK_CUDA(h2d_small(ctx, d_row_off.p, rows->mk_off.data(), (NR + 1) * 8));
  SK_CUDA(h2d_small(ctx, d_col_off.p, cols->mk_off.data(), (NC + 1) * 8));
  DTmp<uint32_t> ra, rb, scol;
  const size_t n_row_entries = tri ? Mc : Mr;
  SK_CUDA(ra.alloc(n_row_entries, ctx)); SK_CUDA(rb.alloc(n_row_entries, ctx)); SK_CUDA(scol.alloc(N, ctx));
  if (N > 0) {
    DTmp<uint64_t> keys, skeys;
    DTmp<uint32_t> vals, svals, eg, head, hscan, rstart, firstq;
    SK_CUDA(keys.alloc(N, ctx)); SK_CUDA(skeys.alloc(N, ctx)); SK_CUDA(vals.alloc(N, ctx)); SK_CUDA(svals.alloc(N, ctx));
    SK_CUDA(eg.alloc(N, ctx)); SK_CUDA(head.alloc(N, ctx)); SK_CUDA(hscan.alloc(N, ctx));
    if (Mc) SK_CUDA(cudaMemcpyAsync(keys.p, cols->markers, Mc * 8, cudaMemcpyDeviceToDevice, st));
    if (Mr) SK_CUDA(cudaMemcpyAsync(keys.p + Mc, rows->markers, Mr * 8, cudaMemcpyDeviceToDevice, st));
    fill_genome_kernel<<<NC, 256, 0, st>>>(d_col_off.p, 0, eg.p); count_launch(ctx);
    if (!tri) { fill_genome_kernel<<<NR, 256, 0, st>>>(d_row_off.p, (uint32_t)Mc, eg.p); count_launch(ctx); }
    iota_kernel<<<div_up64(N, 256), 256, 0, st>>>(vals.p, (uint32_t)N); count_launch(ctx);
    size_t tb = 0;
    SK_CUDA(cub::DeviceRadixSort::SortPairs(nullptr, tb, keys.p, skeys.p, vals.p, svals.p, (int)N, 0, 2 * MARKER_K, st));
    DTmp<uint8_t> tmp;
    SK_CUDA(tmp.alloc(tb, ctx));
    SK_CUDA(cub::DeviceRadixSort::SortPairs(tmp.p, tb, keys.p, skeys.p, vals.p, svals.p, (int)N, 0, 2 * MARKER_K, st));
    run_head_kernel<<<div_up64(N, 256), 256, 0, st>>>(skeys.p, (uint32_t)N, head.p); count_launch(ctx);
    size_t tb2 = 0;
    SK_CUDA(cub::DeviceScan::ExclusiveSum(nullptr, tb2, head.p, hscan.p, N, st));
    DTmp<uint8_t> tmp2;
    SK_CUDA(tmp2.alloc(tb2, ctx));
    SK_CUDA(cub::DeviceScan::ExclusiveSum(tmp2.p, tb2, head.p, hscan.p, N, st));
    uint32_t lh = 0, ls = 0;
    SK_CUDA(cudaMemcpyAsync(&lh, head.p + (N - 1), 4, cudaMemcpyDeviceToHost, st));
    SK_CUDA(cudaMemcpyAsync(&ls, hscan.p + (N - 1), 4, cudaMemcpyDeviceToHost, st));
    SK_CUDA(cudaStreamSynchronize(st));
    const uint32_t n_runs = lh + ls;
    SK_CUDA(rstart.alloc((size_t)n_runs + 1, ctx));
    run_start_kernel<<<div_up64(N, 256), 256, 0, st>>>(head.p, hscan.p, (uint32_t)N, n_runs, rstart.p); count_launch(ctx);
    if (tri) {
      tri_ranges_kernel<<<div_up64(N, 256), 256, 0, st>>>(svals.p, head.p, hscan.p, rstart.p, eg.p, (uint32_t)N, ra.p, rb.p, scol.p);
      count_launch(ctx);
    } else {
      SK_CUDA(firstq.alloc((size_t)n_runs + 1, ctx));
      // runs without query entries never get read; runs without refs: firstq = rstart (empty slice)
      SK_CUDA(cudaMemcpyAsync(firstq.p, rstart.p, ((size_t)n_runs + 1) * 4, cudaMemcpyDeviceToDevice, st));
      qr_firstq_kernel<<<div_up64(N, 256), 256, 0, st>>>(svals.p, head.p, hscan.p, (uint32_t)N, (uint32_t)Mc, firstq.p); count_launch(ctx);
      qr_ranges_kernel<<<div_up64(N, 256), 256, 0, st>>>(svals.p, head.p, hscan.p, rstart.p, firstq.p, eg.p, (uint32_t)N,
                                                        (uint32_t)Mc, ra.p, rb.p, scol.p); count_launch(ctx);
    }
    SK_CUDA(cudaStreamSynchronize(st));
  }
  // ---- row pass with retry on capacity overflow (src/triangle.rs:71: triangle rows 0..N-2)
  return rows_pass(ctx, d_row_off.p, d_col_off.p, tri ? (NR > 0 ? NR - 1 : 0) : NR, NC, ra.p, rb.p, scol.p, mode, mp->rescue_small, cutoff, NR,
                   row_mod, row_rem, out_pairs, out_n);
}

// ------------------------------------------------------------------------------------------------------------------
// Incremental triangle screen (the pipelined sk_triangle screens a GROWING set once per wave): the inverted index is
// kept as ONE sorted array of (marker << 22 | genome).  A wave sorts only its own markers, merges them into the table
// (one streaming pass) and runs only its own genomes as rows: row j finds each of its markers in the table (lower
// bound inside a 16-bit prefix bucket) and walks the run's entries with genome < j.  Same predicate, same pairs as the
// full screen restricted to "larger index in the wave" -- without re-sorting and re-walking everything every wave.
constexpr uint32_t TS_GBITS = 22;                   // genome index bits of a table key (the caller falls back above 2^22 genomes)
constexpr uint32_t TS_PREFIX_BITS = 16;
constexpr uint32_t TS_PREFIX_SHIFT = 2 * MARKER_K + TS_GBITS - TS_PREFIX_BITS;

__global__ void ts_keys_kernel(const uint64_t* __restrict__ markers, const uint64_t* __restrict__ off, uint32_t g_begin,
                               uint64_t* __restrict__ keys) {
  const uint32_t g = g_begin + blockIdx.x;
  const uint64_t base = off[g_begin];
  for (uint64_t i = off[g] + threadIdx.x; i < off[g + 1]; i += blockDim.x) keys[i - base] = (markers[i] << TS_GBITS) | g;
}
// bucket[b] = first table position whose key prefix (key >> shift, 16 bits) is >= b; bucket[2^16] = n
__global__ void ts_bucket_kernel(const uint64_t* __restrict__ key, uint32_t n, uint32_t shift, uint32_t* __restrict__ bucket) {
  const uint32_t b = blockIdx.x * blockDim.x + threadIdx.x;
  if (b > (1u << TS_PREFIX_BITS)) return;
  uint32_t lo = 0, hi = n;
  while (lo < hi) {
    const uint32_t mid = (lo + hi) >> 1;
    if ((key[mid] >> shift) < b) lo = mid + 1; else hi = mid;
  }
  bucket[b] = lo;
}
// One block per NEW genome j (the larger index of its pairs); columns are the genomes i < j.
__global__ void __launch_bounds__(256)
ts_rows_kernel(const uint64_t* __restrict__ markers, const uint64_t* __restrict__ off, const uint64_t* __restrict__ key,
               const uint32_t* __restrict__ bucket, uint32_t g_begin, uint32_t n_genomes, int rescue_small, double cutoff,
               uint32_t tile, uint64_t* __restrict__ pairs, unsigned long long* __restrict__ n_pairs, unsigned long long cap) {
  extern __shared__ uint32_t counts[];
  const uint32_t j = g_begin + blockIdx.x;
  if (j >= n_genomes || j == 0) return;
  const uint64_t mb = off[j], me = off[j + 1];
  const uint64_t card_j = me - mb;
  for (uint32_t t0 = 0; t0 < j; t0 += tile) {
    const uint32_t t1 = min(j, t0 + tile);
    for (uint32_t c = threadIdx.x; c < t1 - t0; c += blockDim.x) counts[c] = 0;
    __syncthreads();
    for (uint64_t e = mb + threadIdx.x; e < me; e += blockDim.x) {
      const uint64_t m = markers[e];
      const uint64_t k0 = m << TS_GBITS;
      const uint32_t b = (uint32_t)(k0 >> TS_PREFIX_SHIFT);
      uint32_t lo = bucket[b], hi = bucket[b + 1];
      while (lo < hi) {
        const uint32_t mid = (lo + hi) >> 1;
        if (key[mid] < k0) lo = mid + 1; else hi = mid;
      }
      // the run of marker m starts at lo; its entries are in ascending genome order, row j's own entry ends the walk
      for (uint32_t t = lo;; t++) {
        const uint64_t kk = key[t];
        const uint32_t col = (uint32_t)(kk & ((1u << TS_GBITS) - 1));
        if ((kk >> TS_GBITS) != m || col >= j) break;
        if (col >= t0 && col < t1) atomicAdd(&counts[col - t0], 1u);
      }
    }
    __syncthreads();
    for (uint32_t c = threadIdx.x; c < t1 - t0; c += blockDim.x) {
      const uint32_t i = t0 + c;
      const uint64_t card_i = off[i + 1] - off[i];
      // screen_refs with the smaller index i as its row (the rescue follows i, src/screen.rs:158-160)
      if (screen_pass(MODE_TRIANGLE, rescue_small, card_i, card_j, counts[c], cutoff)) {
        unsigned long long slot = atomicAdd(n_pairs, 1ull);
        if (slot < cap) pairs[slot] = ((uint64_t)i << 32) | j;
      }
    }
    __syncthreads();
  }
}

struct TriScreen {
  sk_ctx* ctx = nullptr;
  uint64_t* key[2] = {nullptr, nullptr};
  size_t cap = 0, n = 0;
  int cur = 0;
  uint32_t G = 0;
  uint32_t* bucket = nullptr;
};

int tri_screen_create(sk_ctx* ctx, size_t marker_hint, TriScreen** out) {
  TriScreen* t = new TriScreen();
  t->ctx = ctx;
  t->cap = std::max<size_t>(marker_hint, 1024);
  for (int i = 0; i < 2; i++)
    if (ctx->arena.alloc((void**)&t->key[i], t->cap * 8) != cudaSuccess) { tri_screen_free(t); ctx->err = "tri_screen: out of device memory"; return SK_ERR_NOMEM; }
  if (ctx->arena.alloc((void**)&t->bucket, ((1u << TS_PREFIX_BITS) + 2) * 4) != cudaSuccess) { tri_screen_free(t); ctx->err = "tri_screen: out of device memory"; return SK_ERR_NOMEM; }
  *out = t;
  return SK_OK;
}
void tri_screen_free(TriScreen* t) {
  if (!t) return;
  for (int i = 0; i < 2; i++) if (t->key[i]) t->ctx->arena.release(t->key[i]);
  if (t->bucket) t->ctx->arena.release(t->bucket);
  delete t;
}
bool tri_screen_supports(uint32_t n_genomes, uint64_t n_markers) { return n_genomes < (1u << TS_GBITS) && n_markers < (1ull << 31); }

// Adds the markers of the genomes [ts->G, g_end) of `set` to the table and screens the pairs (i, j), i < j, row_begin <= j < g_end
// (`set` must hold the genomes added so far as its prefix).  The pipelined triangle calls it once per wave with row_begin = ts->G;
// a sharded screen (sk_screen_triangle_block) calls it once on an empty table with the rows of one block.
int tri_screen_add(TriScreen* ts, const sk_sketch_set* set, uint32_t g_end, uint32_t row_begin, const sk_map_params* mp,
                   uint64_t** out_pairs, uint64_t* out_n) {
  sk_ctx* ctx = ts->ctx;
  cudaStream_t st = ctx->stream;
  *out_pairs = nullptr; *out_n = 0;
  const uint32_t G = g_end, g_begin = ts->G;
  if (G > set->G || G < g_begin || row_begin < g_begin || row_begin > G || set->mk_off[g_begin] != ts->n || !tri_screen_supports(G, set->mk_off[G])) {
    ctx->err = "tri_screen_add: set does not continue the screened prefix";
    return SK_ERR_PARAM;
  }
  const size_t m_new = set->mk_off[G] - set->mk_off[g_begin], n_tot = ts->n + m_new;
  double screen_val = mp->screen_val == 0. ? 0.80 : mp->screen_val;  // src/triangle.rs:34-42
  const double cutoff = powi21(screen_val);
  if (n_tot > ts->cap) {   // estimate was short: grow both halves, keep the current table
    const size_t ncap = n_tot + n_tot / 2;
    for (int i = 0; i < 2; i++) {
      uint64_t* p = nullptr;
      if (ctx->arena.alloc((void**)&p, ncap * 8) != cudaSuccess) { ctx->err = "tri_screen: out of device memory"; return SK_ERR_NOMEM; }
      if (i == ts->cur && ts->n) SK_CUDA(cudaMemcpyAsync(p, ts->key[i], ts->n * 8, cudaMemcpyDeviceToDevice, st));
      SK_CUDA(cudaStreamSynchronize(st));
      ctx->arena.release(ts->key[i]);
      ts->key[i] = p;
    }
    ts->cap = ncap;
  }
  DTmp<uint64_t> d_off;
  SK_CUDA(d_off.alloc((size_t)G + 1, ctx));
  SK_CUDA(h2d_small(ctx, d_off.p, set->mk_off.data(), ((size_t)G + 1) * 8));
  if (m_new > 0) {
    DTmp<uint64_t> nk, snk;
    SK_CUDA(nk.alloc(m_new, ctx)); SK_CUDA(snk.alloc(m_new, ctx));
    ts_keys_kernel<<<G - g_begin, 256, 0, st>>>(set->markers, d_off.p, g_begin, nk.p); count_launch(ctx);
    // stable sort on the marker bits only: inside a run the genomes stay ascending (they are laid out genome-major)
    size_t tb = 0;
    SK_CUDA(cub::DeviceRadixSort::SortKeys(nullptr, tb, nk.p, snk.p, (int)m_new, (int)TS_GBITS, (int)(TS_GBITS + 2 * MARKER_K), st));
    DTmp<uint8_t> tmp;
    SK_CUDA(tmp.alloc(tb, ctx));
    SK_CUDA(cub::DeviceRadixSort::SortKeys(tmp.p, tb, nk.p, snk.p, (int)m_new, (int)TS_GBITS, (int)(TS_GBITS + 2 * MARKER_K), st));
    if (ts->n == 0) {
      SK_CUDA(cudaMemcpyAsync(ts->key[1 - ts->cur], snk.p, m_new * 8, cudaMemcpyDeviceToDevice, st));
    } else {       // keys are distinct (marker, genome) pairs, so the unstable merge has one possible output
      size_t mb = 0;
      SK_CUDA(cub::DeviceMerge::MergeKeys(nullptr, mb, ts->key[ts->cur], (int)ts->n, snk.p, (int)m_new, ts->key[1 - ts->cur], ::cuda::std::less<uint64_t>{}, st));
      DTmp<uint8_t> tmp2;
      SK_CUDA(tmp2.alloc(mb, ctx));
      SK_CUDA(cub::DeviceMerge::MergeKeys(tmp2.p, mb, ts->key[ts->cur], (int)ts->n, snk.p, (int)m_new, ts->key[1 - ts->cur], ::cuda::std::less<uint64_t>{}, st));
      count_launch(ctx);
    }
    ts->cur = 1 - ts->cur;
    SK_CUDA(cudaStreamSynchronize(st));   // temporaries go back to the arena below
  }
  ts->n = n_tot; ts->G = G;
  uint64_t* host = nullptr;
  unsigned long long n = 0;
  if (G > row_begin && G > 1) {
    // (a row's walk always ends at its own table entry, so it never runs past the end of the table)
    ts_bucket_kernel<<<((1u << TS_PREFIX_BITS) + 256) / 256, 256, 0, st>>>(ts->key[ts->cur], (uint32_t)n_tot, TS_PREFIX_SHIFT, ts->bucket); count_launch(ctx);
    const uint32_t tile = std::min<uint32_t>(std::max<uint32_t>(G, 1), 48 * 1024);
    const size_t smem = (size_t)tile * 4;
    SK_CUDA(cudaFuncSetAttribute(ts_rows_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 48 * 1024 * 4));   // constant: see run_screen
    unsigned long long cap = std::max<unsigned long long>(1ull << 20, 64ull * (G - row_begin));
    DTmp<unsigned long long> d_n;
    SK_CUDA(d_n.alloc(1, ctx));
    DTmp<uint64_t> d_pairs;
    for (int attempt = 0; attempt < 2; attempt++) {
      SK_CUDA(d_pairs.alloc(cap, ctx));
      SK_CUDA(cudaMemsetAsync(d_n.p, 0, 8, st));
      SK_LAUNCH(ctx, "screen_rows_kernel", (ts_rows_kernel<<<G - row_begin, 256, smem, st>>>(
          set->markers, d_off.p, ts->key[ts->cur], ts->bucket, row_begin, G, mp->rescue_small, cutoff, tile, d_pairs.p, d_n.p, cap)));
      SK_CUDA(cudaMemcpyAsync(&n, d_n.p, 8, cudaMemcpyDeviceToHost, st));
      SK_CUDA(cudaStreamSynchronize(st));
      SK_CUDA(cudaGetLastError());
      if (n <= cap) break;
      cap = n;
    }
    host = (uint64_t*)malloc(std::max<size_t>(n, 1) * 8);
    if (!host) return SK_ERR_NOMEM;
    if (n > 0) {
      DTmp<uint64_t> sorted;
      SK_CUDA(sorted.alloc(n, ctx));
      size_t tb = 0;
      SK_CUDA(cub::DeviceRadixSort::SortKeys(nullptr, tb, d_pairs.p, sorted.p, (uint64_t)n, 0, 64, st));
      DTmp<uint8_t> tmp;
      SK_CUDA(tmp.alloc(tb, ctx));
      SK_CUDA(cub::DeviceRadixSort::SortKeys(tmp.p, tb, d_pairs.p, sorted.p, (uint64_t)n, 0, 64, st));
      SK_CUDA(cudaMemcpyAsync(host, sorted.p, n * 8, cudaMemcpyDeviceToHost, st));
      SK_CUDA(cudaStreamSynchronize(st));
    }
  } else {
    host = (uint64_t*)malloc(8);
    if (!host) return SK_ERR_NOMEM;
  }
  *out_pairs = host;
  *out_n = n;
  return SK_OK;
}

// ------------------------------------------------------------------------------------------------------------------
// Persistent reference marker index (search: many query groups against one database).  The query x ref screen of
// run_screen sorts the reference and query markers together for every call; here the reference markers are sorted ONCE,
// per contiguous part of the references, into (marker, local reference) entries -- a stable sort of the genome-major
// markers, so a run's entries stay in reference order exactly as inside run_screen's runs -- with a 16-bit prefix bucket
// table.  A query group then only looks each of its markers up (ri_lookup_kernel writes the run's slice as ra / rb, as
// qr_ranges_kernel does) and runs the same screen_rows_kernel and pair sort as run_screen, once per part.
constexpr uint32_t RI_PREFIX_SHIFT = 2 * MARKER_K - TS_PREFIX_BITS;

// entry i of the part [r0, r0 + gridDim.x) of a genome-major set belongs to local reference blockIdx.x
__global__ void ri_part_ref_kernel(const uint64_t* __restrict__ off, uint32_t r0, uint32_t* __restrict__ ref) {
  const uint32_t g = r0 + blockIdx.x;
  const uint64_t base = off[r0];
  for (uint64_t i = off[g] + threadIdx.x; i < off[g + 1]; i += blockDim.x) ref[i - base] = blockIdx.x;
}
// query marker e -> the slice [ra[e], rb[e]) of the part's sorted keys that holds the same marker (empty when none does)
__global__ void __launch_bounds__(256)
ri_lookup_kernel(const uint64_t* __restrict__ markers, uint64_t n_markers, const uint64_t* __restrict__ key,
                 const uint32_t* __restrict__ bucket, uint32_t* __restrict__ ra, uint32_t* __restrict__ rb) {
  for (uint64_t e = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; e < n_markers; e += (uint64_t)gridDim.x * blockDim.x) {
    const uint64_t m = markers[e];
    const uint64_t b = m >> RI_PREFIX_SHIFT;
    uint32_t lo = 0, hi = 0;
    if (b < (1u << TS_PREFIX_BITS)) {      // markers are < 2^42 (import refuses larger ones): every prefix has a bucket
      const uint32_t end = bucket[b + 1];
      lo = bucket[b];
      hi = end;
      while (lo < hi) {                    // first key >= m
        const uint32_t mid = (lo + hi) >> 1;
        if (key[mid] < m) lo = mid + 1; else hi = mid;
      }
      hi = end;
      uint32_t l2 = lo;
      while (l2 < hi) {                    // first key > m (a larger marker of the next prefix starts at bucket[b + 1])
        const uint32_t mid = (l2 + hi) >> 1;
        if (key[mid] <= m) l2 = mid + 1; else hi = mid;
      }
      hi = l2;
    }
    ra[e] = lo;
    rb[e] = hi;
  }
}

struct RefIndexPart {
  uint32_t r0 = 0, r1 = 0;        // references [r0, r1)
  size_t n = 0;                   // entries = their markers
  uint64_t* key = nullptr;        // [n] markers, sorted
  uint32_t* scol = nullptr;       // [n] local reference (r - r0) of each sorted entry
  uint32_t* bucket = nullptr;     // [2^16 + 1] first entry of each 16-bit marker prefix
};

// entries per part: < 2^31 (cub's item count, and the 32-bit ra / rb slices of screen_rows_kernel).  SK_REF_INDEX_PART_MARKERS
// lowers it (a test hook: many parts from a small database); read when an index is created.
static size_t ref_index_part_limit() {
  size_t lim = (1ull << 31) - 1;
  if (const char* e = getenv("SK_REF_INDEX_PART_MARKERS")) lim = std::min<size_t>(lim, (size_t)std::max(1ll, atoll(e)));
  return lim;
}

}  // namespace sk

struct sk_ref_index {
  sk_ctx* ctx = nullptr;
  uint32_t G = 0;
  uint64_t* col_off = nullptr;    // [G + 1] device copy of the references' marker offsets
  std::vector<sk::RefIndexPart> parts;
  size_t bytes = 0;               // device bytes held
};

namespace sk {

static void ref_index_release(sk_ref_index* x) {
  if (!x) return;
  for (auto& p : x->parts) {
    if (p.key) x->ctx->arena.release(p.key);
    if (p.scol) x->ctx->arena.release(p.scol);
    if (p.bucket) x->ctx->arena.release(p.bucket);
  }
  if (x->col_off) x->ctx->arena.release(x->col_off);
  delete x;
}

// the parts of x (ctx, G set) from refs; on failure the caller releases x
static int ref_index_build(sk_ctx* ctx, const sk_sketch_set* refs, sk_ref_index* x) {
  cudaStream_t st = ctx->stream;
  auto fail = [&](const char* msg) { ctx->err = msg; return SK_ERR_NOMEM; };
  const auto alloc = [&](void** p, size_t bytes) { x->bytes += bytes; return ctx->arena.alloc(p, std::max<size_t>(bytes, 8)); };
  if (alloc((void**)&x->col_off, ((size_t)x->G + 1) * 8) != cudaSuccess) return fail("ref_index: out of device memory");
  SK_CUDA(h2d_small(ctx, x->col_off, refs->mk_off.data(), ((size_t)x->G + 1) * 8));
  const size_t lim = ref_index_part_limit();
  for (uint32_t r0 = 0; r0 < x->G;) {
    uint32_t r1 = r0 + 1;     // at least one reference; a genome holds far fewer than 2^31 markers
    while (r1 < x->G && refs->mk_off[r1 + 1] - refs->mk_off[r0] <= lim) r1++;
    RefIndexPart p;
    p.r0 = r0; p.r1 = r1;
    p.n = refs->mk_off[r1] - refs->mk_off[r0];
    x->parts.push_back(p);
    RefIndexPart& q = x->parts.back();
    if (alloc((void**)&q.key, q.n * 8) != cudaSuccess || alloc((void**)&q.scol, q.n * 4) != cudaSuccess ||
        alloc((void**)&q.bucket, ((1u << TS_PREFIX_BITS) + 1) * 4) != cudaSuccess)
      return fail("ref_index: out of device memory");
    if (q.n > 0) {
      DTmp<uint32_t> ref;
      SK_CUDA(ref.alloc(q.n, ctx));
      ri_part_ref_kernel<<<r1 - r0, 256, 0, st>>>(x->col_off, r0, ref.p); count_launch(ctx);
      // stable on the marker bits: inside a run the references stay ascending (the set is genome-major), as in run_screen
      size_t tb = 0;
      const uint64_t* in = refs->markers + refs->mk_off[r0];
      SK_CUDA(cub::DeviceRadixSort::SortPairs(nullptr, tb, in, q.key, ref.p, q.scol, (int)q.n, 0, 2 * MARKER_K, st));
      DTmp<uint8_t> tmp;
      SK_CUDA(tmp.alloc(tb, ctx));
      SK_CUDA(cub::DeviceRadixSort::SortPairs(tmp.p, tb, in, q.key, ref.p, q.scol, (int)q.n, 0, 2 * MARKER_K, st));
    }
    ts_bucket_kernel<<<((1u << TS_PREFIX_BITS) + 256) / 256, 256, 0, st>>>(q.key, (uint32_t)q.n, RI_PREFIX_SHIFT, q.bucket); count_launch(ctx);
    SK_CUDA(cudaStreamSynchronize(st));   // the temporaries go back to the arena
    r0 = r1;
  }
  SK_CUDA(cudaGetLastError());
  return SK_OK;
}

static int ref_index_create(sk_ctx* ctx, const sk_sketch_set* refs, sk_ref_index** out) {
  sk_ref_index* x = new sk_ref_index();
  x->ctx = ctx;
  x->G = refs->G;
  const int rc = ref_index_build(ctx, refs, x);
  if (rc != SK_OK) { ref_index_release(x); return rc; }
  *out = x;
  return SK_OK;
}

static int ref_index_screen(sk_ctx* ctx, const sk_ref_index* x, const sk_sketch_set* queries, const sk_map_params* mp, int mode,
                            uint64_t** out_pairs, uint64_t* out_n) {
  cudaStream_t st = ctx->stream;
  const uint32_t NR = queries->G;
  *out_pairs = nullptr; *out_n = 0;
  if (NR == 0 || x->G == 0) { *out_pairs = (uint64_t*)malloc(8); return *out_pairs ? SK_OK : SK_ERR_NOMEM; }
  const double cutoff = powi21(mp->screen_val == 0. ? 0.80 : mp->screen_val);   // src/dist.rs:68-77
  const size_t Mr = queries->M;
  DTmp<uint64_t> d_row_off;
  SK_CUDA(d_row_off.alloc((size_t)NR + 1, ctx));
  SK_CUDA(h2d_small(ctx, d_row_off.p, queries->mk_off.data(), ((size_t)NR + 1) * 8));
  DTmp<uint32_t> ra, rb;
  SK_CUDA(ra.alloc(Mr, ctx)); SK_CUDA(rb.alloc(Mr, ctx));
  std::vector<uint64_t> all;
  for (const RefIndexPart& p : x->parts) {
    if (Mr) {
      const uint32_t blocks = (uint32_t)std::min<uint64_t>((Mr + 255) / 256, 1u << 20);
      ri_lookup_kernel<<<blocks, 256, 0, st>>>(queries->markers, Mr, p.key, p.bucket, ra.p, rb.p); count_launch(ctx);
    }
    uint64_t* pairs = nullptr; uint64_t n = 0;
    SK_TRY(rows_pass(ctx, d_row_off.p, x->col_off + p.r0, NR, p.r1 - p.r0, ra.p, rb.p, p.scol, mode, mp->rescue_small, cutoff, NR, 1, 0,
                     &pairs, &n));
    // pairs are (local ref << 32 | query), sorted; parts ascend, so the concatenation stays sorted
    const uint64_t shift = (uint64_t)p.r0 << 32;
    if (x->parts.size() == 1) { *out_pairs = pairs; *out_n = n; return SK_OK; }
    for (uint64_t i = 0; i < n; i++) all.push_back(pairs[i] + shift);
    free(pairs);
  }
  uint64_t* host = (uint64_t*)malloc(std::max<size_t>(all.size(), 1) * 8);
  if (!host) return SK_ERR_NOMEM;
  if (!all.empty()) memcpy(host, all.data(), all.size() * 8);
  *out_pairs = host;
  *out_n = all.size();
  return SK_OK;
}

}  // namespace sk

extern "C" {

int sk_screen_triangle(sk_ctx* ctx, const sk_sketch_set* set, const sk_map_params* mp, uint64_t** pairs, uint64_t* n) {
  if (!ctx || !set || !mp || !pairs || !n) return SK_ERR_PARAM;
  SK_CUDA(cudaSetDevice(ctx->device));
  return sk::run_screen(ctx, set, set, sk::MODE_TRIANGLE, mp, pairs, n);
}

int sk_screen_triangle_rows(sk_ctx* ctx, const sk_sketch_set* set, const sk_map_params* mp, uint32_t row_mod, uint32_t row_rem,
                            uint64_t** pairs, uint64_t* n) {
  if (!ctx || !set || !mp || !pairs || !n || row_mod == 0 || row_rem >= row_mod) return SK_ERR_PARAM;
  SK_CUDA(cudaSetDevice(ctx->device));
  return sk::run_screen(ctx, set, set, sk::MODE_TRIANGLE, mp, pairs, n, row_mod, row_rem);
}

int sk_screen_triangle_block(sk_ctx* ctx, const sk_sketch_set* set, uint32_t g_begin, uint32_t g_end, const sk_map_params* mp,
                             uint64_t** pairs, uint64_t* n) {
  if (!ctx || !set || !mp || !pairs || !n || g_begin > g_end || g_end > set->G) return SK_ERR_PARAM;
  SK_CUDA(cudaSetDevice(ctx->device));
  if (!sk::tri_screen_supports(g_end, set->mk_off[g_end]) || getenv("SK_FULL_RESCREEN")) {   // one-shot screen of everything, then the block's rows
    uint64_t* all = nullptr; uint64_t na = 0;
    SK_TRY(sk::run_screen(ctx, set, set, sk::MODE_TRIANGLE, mp, &all, &na));
    uint64_t m = 0;
    for (uint64_t i = 0; i < na; i++) { const uint32_t j = (uint32_t)all[i]; if (j >= g_begin && j < g_end) all[m++] = all[i]; }
    *pairs = all; *n = m;
    return SK_OK;
  }
  sk::TriScreen* ts = nullptr;
  SK_TRY(sk::tri_screen_create(ctx, set->mk_off[g_end] + 1024, &ts));
  const int rc = sk::tri_screen_add(ts, set, g_end, g_begin, mp, pairs, n);
  sk::tri_screen_free(ts);
  return rc;
}

int sk_screen_query_ref(sk_ctx* ctx, const sk_sketch_set* refs, const sk_sketch_set* queries, const sk_map_params* mp, int mode,
                        uint64_t** pairs, uint64_t* n) {
  if (!ctx || !refs || !queries || !mp || !pairs || !n || mode < 0 || mode > 3) return SK_ERR_PARAM;
  SK_CUDA(cudaSetDevice(ctx->device));
  return sk::run_screen(ctx, queries, refs, mode, mp, pairs, n);
}

int sk_ref_index_create(sk_ctx* ctx, const sk_sketch_set* refs, sk_ref_index** idx) {
  if (!ctx || !refs || !idx) return SK_ERR_PARAM;
  *idx = nullptr;
  if (refs->ctx != ctx) { ctx->err = "sk_ref_index_create: the set lives on another context"; return SK_ERR_PARAM; }
  SK_CUDA(cudaSetDevice(ctx->device));
  return sk::ref_index_create(ctx, refs, idx);
}

int sk_ref_index_screen(sk_ctx* ctx, const sk_ref_index* idx, const sk_sketch_set* queries, const sk_map_params* mp, int mode,
                        uint64_t** pairs, uint64_t* n) {
  if (!ctx || !idx || !queries || !mp || !pairs || !n || mode < 0 || mode > 3) return SK_ERR_PARAM;
  if (idx->ctx != ctx || queries->ctx != ctx) { ctx->err = "sk_ref_index_screen: the index and the queries must live on ctx"; return SK_ERR_PARAM; }
  SK_CUDA(cudaSetDevice(ctx->device));
  return sk::ref_index_screen(ctx, idx, queries, mp, mode, pairs, n);
}

int sk_ref_index_info(const sk_ref_index* idx, uint32_t* n_refs, uint32_t* n_parts, uint64_t* device_bytes) {
  if (!idx) return SK_ERR_PARAM;
  if (n_refs) *n_refs = idx->G;
  if (n_parts) *n_parts = (uint32_t)idx->parts.size();
  if (device_bytes) *device_bytes = idx->bytes;
  return SK_OK;
}

int sk_ref_index_free(sk_ref_index* idx) {
  if (!idx) return SK_OK;
  sk_ctx* ctx = idx->ctx;
  SK_CUDA(cudaSetDevice(ctx->device));
  sk::ref_index_release(idx);
  return SK_OK;
}

}  // extern "C"
