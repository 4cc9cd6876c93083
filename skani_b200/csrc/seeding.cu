// seeding.cu -- FracMinHash seeding + sketch assembly on the device (sm_90a).
//
// Replaces avx2_seeding::avx2_fmh_seeds (reference src/avx2_seeding.rs:33-272), Sketch::add_seed_position
// (src/types.rs:281-304) and the per-file assembly of file_io::fastx_to_sketches (src/file_io.rs:141-252).
//
// Pipeline for one sub-batch of contigs (all arrays device resident):
//   pack_kernel     ASCII -> 2-bit units (u64 per 32 bases) + 'N' bitmask (u32 per 32 bases)        [HBM bound: 1.4 B/base]
//   hashpass_kernel per unit: 32 windows -> seed k-mer -> mm_hash64 -> 32-bit pass mask + popcount  [integer-ALU bound]
//   (cub) exclusive scan of popcounts -> record offsets in (genome, contig, pos) order
//   expand_kernel   per set bit: (kmer, pos, contig<<1|canonical) record + canonical 21-mer marker for hash < T_marker
//   build_views     k-mer-ordered view (segmented radix sort per genome), distinct k-mer groups, multiplicities,
//                   marker sort + dedup per genome  (the flat-array equivalent of the reference's HashMap/HashSet)
#include <cub/cub.cuh>
#include <thrust/iterator/transform_iterator.h>

#include <algorithm>
#include <cstdlib>
#include <cstring>

#include "sk_core.cuh"
#include "sk_internal.h"

namespace sk {

uint64_t count_launch(sk_ctx* ctx, uint64_t n) {
  ctx->launches += n;
  return ctx->launches;
}

// ------------------------------------------------------------------------------------------------------------
// kernels
// ------------------------------------------------------------------------------------------------------------
constexpr int PACK_THREADS = 256;
constexpr uint32_t UCOARSE_SHIFT = 8;   // host-built index: contig of every 256th unit (4 B per 8 KB of sequence)

// contig lookup for a unit: narrowed binary search over the unit prefix offsets
__device__ __forceinline__ uint32_t find_contig(const uint32_t* __restrict__ cuoff, uint32_t u, uint32_t lo_hint, uint32_t hi_hint) {
  uint32_t lo = lo_hint, hi = hi_hint;  // invariant: cuoff[lo] <= u < cuoff[hi]
  while (hi - lo > 1) {
    uint32_t mid = (lo + hi) >> 1;
    if (cuoff[mid] <= u) lo = mid; else hi = mid;
  }
  return lo;
}
// contig of unit u through the coarse index (ucoarse has (n_units >> 8) + 2 entries, the last = n_contigs - 1): at most a
// handful of contig starts fall inside one 256-unit stretch, so the search is 0-3 steps on cached data
__device__ __forceinline__ uint32_t contig_of_unit(const uint32_t* __restrict__ ucoarse, const uint32_t* __restrict__ cuoff, uint32_t u) {
  const uint32_t lo = __ldg(ucoarse + (u >> UCOARSE_SHIFT)), hi = __ldg(ucoarse + (u >> UCOARSE_SHIFT) + 1) + 1;
  return find_contig(cuoff, u, lo, hi);
}

// ASCII -> 2-bit units + N mask for the units [u_begin, n_units) of a sub-batch (the units before u_begin arrived packed
// from the host).  Thread per unit, nine aligned 32-bit loads realigned with funnel shifts (contig starts are arbitrary
// byte offsets), then SIMD-in-register conversion: no shared-memory table.
__global__ void __launch_bounds__(PACK_THREADS)
pack_kernel(const uint8_t* __restrict__ ascii, const uint64_t* __restrict__ coff, const uint32_t* __restrict__ cuoff,
            const uint32_t* __restrict__ clen, const uint32_t* __restrict__ ucoarse, uint32_t u_begin, uint32_t n_units,
            uint64_t* __restrict__ P, uint32_t* __restrict__ NM, int small_n) {
  const uint32_t u = u_begin + blockIdx.x * PACK_THREADS + threadIdx.x;
  if (u >= n_units) return;
  const uint32_t ci = contig_of_unit(ucoarse, cuoff, u);
  const uint32_t ul = u - cuoff[ci];
  const uint32_t len = clen[ci];
  const uint32_t nvalid = min(32u, len - 32u * ul);
  const uint8_t* src = ascii + coff[ci] + 32ull * ul;
  const uintptr_t addr = (uintptr_t)src;
  const uint32_t* wp = (const uint32_t*)(addr & ~(uintptr_t)3);
  const uint32_t sh = (uint32_t)(addr & 3) * 8;
  const uint32_t nwords = (nvalid + (uint32_t)(addr & 3) + 3) >> 2;  // words overlapping the valid span
  uint32_t w[9];
#pragma unroll
  for (int i = 0; i < 9; i++) w[i] = (i < (int)nwords) ? __ldg(wp + i) : 0u;
  uint64_t packed = 0;
  uint32_t nm = 0;
#pragma unroll
  for (int i = 0; i < 8; i++) {
    const uint32_t r = __funnelshift_r(w[i], w[i + 1], sh);
    uint32_t c8, n4;
    pack_word(r, c8, n4, small_n != 0);
    packed |= (uint64_t)c8 << (8 * i);
    nm |= n4 << (4 * i);
  }
  if (nvalid < 32u) { packed &= (1ull << (2 * nvalid)) - 1ull; nm &= (1u << nvalid) - 1u; }   // bases past the contig end read as 0
  P[u] = packed;
  NM[u] = nm;
}

constexpr int HASH_THREADS = 128;

// ---- A/B variants of the hash arithmetic (SK_HASHPASS_VARIANT=1|2): the kernel is bound
// by the ALU pipe (LOP3 / SHF / IADD3) while the FMA pipe (IMAD) has headroom, so the right shifts of the three xor-shift
// steps can be issued as multiplications: x >> s == mul.hi(x, 2^(32-s)).  The multipliers arrive as kernel arguments so
// that ptxas cannot turn them back into shifts.  V=1: the high word only; V=2: both words (low word = mul.hi(lo, c) + hi * c).
template <int V>
__device__ __forceinline__ uint64_t xorshift_var(uint64_t key, uint32_t s, uint32_t c) {
  const uint32_t lo = (uint32_t)key, hi = (uint32_t)(key >> 32);
  uint32_t hs, ls;
  asm("mul.hi.u32 %0, %1, %2;" : "=r"(hs) : "r"(hi), "r"(c));
  if (V == 1) ls = __funnelshift_r(lo, hi, s);
  else { uint32_t t; asm("mul.hi.u32 %0, %1, %2;" : "=r"(t) : "r"(lo), "r"(c)); ls = t + hi * c; }
  return ((uint64_t)(hi ^ hs) << 32) | (uint64_t)(lo ^ ls);
}
template <int V>
__device__ __forceinline__ uint32_t unit_pass_mask_var(uint64_t lo, uint64_t hi, uint32_t nm_lo, uint32_t nm_hi, uint32_t n, uint32_t ul,
                                                       uint32_t seed_mask32, uint64_t threshold, uint32_t c24, uint32_t c14, uint32_t c28) {
  const uint32_t valid = unit_valid_mask(n, ul);
  if (valid == 0) return 0;
  const uint64_t clo = ~lo, chi = ~hi;
  const uint64_t tlo = pair_reverse64(hi), thi = pair_reverse64(lo);
  const uint32_t c[4] = {(uint32_t)clo, (uint32_t)(clo >> 32), (uint32_t)chi, (uint32_t)(chi >> 32)};
  const uint32_t t[4] = {(uint32_t)tlo, (uint32_t)(tlo >> 32), (uint32_t)thi, (uint32_t)(thi >> 32)};
  uint32_t pass = 0;
#pragma unroll
  for (uint32_t j = 0; j < 32; j++) {
    const uint32_t orv = 24 + 2 * j, ofw = 62 - 2 * j;
    const uint32_t rs = funnel_r32(c[orv >> 5], c[(orv >> 5) + 1], orv & 31) & seed_mask32;
    const uint32_t fs = funnel_r32(t[ofw >> 5], t[(ofw >> 5) + 1], ofw & 31) & seed_mask32;
    const uint32_t seed = fs < rs ? fs : rs;
    uint64_t key = ~((uint64_t)seed * 0x200001ull);
    key = xorshift_var<V>(key, 24, c24);
    key = key * 265ull;
    key = xorshift_var<V>(key, 14, c14);
    key = key * 21ull;
    key = xorshift_var<V>(key, 28, c28);
    key = key * 0x80000001ull;
    if (key < threshold) pass |= 1u << j;
  }
  pass &= valid;
  if ((nm_lo | nm_hi) != 0 && pass != 0) pass &= ~unit_n_suppress_mask(n, ul, nm_lo, nm_hi, pass);
  return pass;
}

template <int V>
__global__ void __launch_bounds__(HASH_THREADS)
hashpass_kernel(const uint64_t* __restrict__ P, const uint32_t* __restrict__ NM, const uint32_t* __restrict__ ucoarse,
                const uint32_t* __restrict__ cuoff, const uint32_t* __restrict__ clen, uint32_t n_units,
                uint64_t seed_mask, uint64_t threshold, uint32_t* __restrict__ PM, uint32_t c24, uint32_t c14, uint32_t c28,
                uint32_t scalar_k) {
  uint32_t u = blockIdx.x * HASH_THREADS + threadIdx.x;
  if (u >= n_units) return;
  // the unit loads do not wait for the contig lookup (ucoarse -> cuoff / clen is a two-level dependent chain): the previous
  // unit is fetched unconditionally and dropped afterwards if this unit turns out to be the first of its contig
  const uint64_t hi = P[u];
  const uint64_t lo_raw = u ? P[u - 1] : 0ull;
  const uint32_t nhi = NM[u];
  const uint32_t nlo_raw = u ? NM[u - 1] : 0u;
  const uint32_t ci = contig_of_unit(ucoarse, cuoff, u);
  const uint32_t ul = u - cuoff[ci];
  const uint32_t n = clen[ci];
  const uint64_t lo = ul ? lo_raw : 0ull;
  const uint32_t nlo = ul ? nlo_raw : 0u;
  if (V == 0) PM[u] = unit_pass_mask_fast(lo, hi, nlo, nhi, n, ul, (uint32_t)seed_mask, threshold, scalar_k);
  else PM[u] = unit_pass_mask_var<V>(lo, hi, nlo, nhi, n, ul, (uint32_t)seed_mask, threshold, c24, c14, c28);
}

// one thread per unit with a non-empty pass mask: regenerate the few passing windows and emit their records
__global__ void __launch_bounds__(256)
expand_kernel(const uint64_t* __restrict__ P, const uint32_t* __restrict__ ucoarse, const uint32_t* __restrict__ cuoff,
              const uint32_t* __restrict__ clocal, uint32_t n_units, const uint32_t* __restrict__ PM,
              const uint32_t* __restrict__ uoff, uint64_t seed_mask, uint64_t threshold_marker,
              uint32_t* __restrict__ pv_kmer, uint32_t* __restrict__ pv_pos, uint32_t* __restrict__ pv_cc,
              uint64_t* __restrict__ mkv) {
  uint32_t u = blockIdx.x * 256 + threadIdx.x;
  if (u >= n_units) return;
  uint32_t pass = PM[u];
  if (pass == 0) return;
  uint32_t ci = contig_of_unit(ucoarse, cuoff, u);
  uint32_t ul = u - cuoff[ci];
  uint64_t hi = P[u];
  uint64_t lo = ul ? P[u - 1] : 0ull;
  WindowCtx w = make_window_ctx(lo, hi);
  uint32_t o = uoff[u];
  uint32_t cl = clocal[ci];
  while (pass) {
    uint32_t j = __ffs(pass) - 1;
    pass &= pass - 1;
    bool canon;
    uint32_t seed = window_seed(w, j, seed_mask, &canon);
    pv_kmer[o] = seed;
    pv_pos[o] = 32u * ul + j;                       // index of the window's last base (src/avx2_seeding.rs:184,207)
    pv_cc[o] = (cl << 1) | (canon ? 1u : 0u);       // SeedPosition::new (src/types.rs:135-143)
    // marker gated by the SEED's hash (src/avx2_seeding.rs:197)
    mkv[o] = (mm_hash64(seed) < threshold_marker) ? window_marker(w, j) : ~0ull;
    o++;
  }
}

__global__ void gather_u32_kernel(const uint32_t* __restrict__ src, const uint32_t* __restrict__ idx, uint32_t n,
                                  uint32_t src_len, uint32_t total, uint32_t* __restrict__ dst) {
  uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  uint32_t k = idx[i];
  dst[i] = (k >= src_len) ? total : src[k];
}

// same, the value for "one past the end" taken from the device: last element + its own count (the popcount of the last pass
// mask, or the last flag) -- the host does not have to know the total before this kernel is queued
__global__ void gather_u32_tail_kernel(const uint32_t* __restrict__ src, const uint32_t* __restrict__ idx, uint32_t n,
                                       uint32_t src_len, const uint32_t* __restrict__ tail, int tail_is_mask,
                                       uint32_t* __restrict__ dst) {
  uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  uint32_t k = idx[i];
  if (k >= src_len) { const uint32_t t = tail[src_len - 1]; dst[i] = src[src_len - 1] + (tail_is_mask ? (uint32_t)__popc(t) : t); }
  else dst[i] = src[k];
}

__global__ void marker_flag_kernel(const uint64_t* __restrict__ mkv, uint32_t n, uint32_t* __restrict__ flag) {
  uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) flag[i] = (mkv[i] != ~0ull) ? 1u : 0u;
}
__global__ void marker_scatter_kernel(const uint64_t* __restrict__ mkv, const uint32_t* __restrict__ scan, uint32_t n,
                                      uint64_t* __restrict__ out) {
  uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n && mkv[i] != ~0ull) out[scan[i]] = mkv[i];
}

// ---- view building (block per genome) ------------------------------------------------------------------
__global__ void iota_local_kernel(const uint64_t* __restrict__ seg_off, uint32_t* __restrict__ vals) {
  uint32_t g = blockIdx.x;
  uint64_t b = seg_off[g], e = seg_off[g + 1];
  for (uint64_t i = b + (uint64_t)blockIdx.y * blockDim.x + threadIdx.x; i < e; i += (uint64_t)blockDim.x * gridDim.y) vals[i] = (uint32_t)(i - b);
}

// sort keys of the k-mer view: (genome << kbits | k-mer), value = the record's index inside its genome.  ONE device-wide radix
// sort of these keys orders every genome of the sub-batch by (kmer, contig, pos) at once (stable), instead of a segmented
// sort that runs one block per genome and pass
//
// When genome, k-mer and the record's index inside its genome fit 64 bits together (ibits > 0: always, short of sub-batches of
// thousands of multi-Gbp genomes) the index rides in the LOW bits of the key and the sort is keys-only over the bits above it:
// 16 instead of 24 bytes moved per record and pass, no value arrays.
__global__ void kview_keys_kernel(const uint64_t* __restrict__ seg_off, const uint32_t* __restrict__ pv_kmer, uint32_t kbits,
                                  uint32_t ibits, uint64_t* __restrict__ keys, uint32_t* __restrict__ vals) {
  const uint32_t g = blockIdx.x;
  const uint64_t b = seg_off[g], e = seg_off[g + 1];
  for (uint64_t i = b + (uint64_t)blockIdx.y * blockDim.x + threadIdx.x; i < e; i += (uint64_t)blockDim.x * gridDim.y) {
    const uint64_t k = ((uint64_t)g << kbits) | pv_kmer[i];
    if (ibits) keys[i] = (k << ibits) | (uint64_t)(i - b);
    else { keys[i] = k; vals[i] = (uint32_t)(i - b); }
  }
}
__global__ void marker_keys_kernel(const uint64_t* __restrict__ seg_off, uint64_t* __restrict__ mk) {   // in place: genome << 42 | marker
  const uint32_t g = blockIdx.x;
  const uint64_t b = seg_off[g], e = seg_off[g + 1];
  for (uint64_t i = b + (uint64_t)blockIdx.y * blockDim.x + threadIdx.x; i < e; i += (uint64_t)blockDim.x * gridDim.y) mk[i] |= (uint64_t)g << (2 * MARKER_K);
}

// after the sort by k-mer: gather the k-mer view and flag group heads
__global__ void kview_gather_kernel(const uint64_t* __restrict__ seg_off, const uint64_t* __restrict__ skmer,
                                    const uint32_t* __restrict__ perm, const uint32_t* __restrict__ pv_pos,
                                    const uint32_t* __restrict__ pv_cc, uint32_t* __restrict__ kv_pos,
                                    uint32_t* __restrict__ kv_cc, uint32_t* __restrict__ head, uint32_t ibits) {
  uint32_t g = blockIdx.x;
  uint64_t b = seg_off[g], e = seg_off[g + 1];
  const uint64_t imask = (1ull << ibits) - 1;
  for (uint64_t i = b + (uint64_t)blockIdx.y * blockDim.x + threadIdx.x; i < e; i += (uint64_t)blockDim.x * gridDim.y) {
    const uint64_t k = skmer[i];
    uint32_t r = ibits ? (uint32_t)(k & imask) : perm[i];
    kv_pos[i] = pv_pos[b + r];
    kv_cc[i] = pv_cc[b + r];
    head[i] = (i == b || (k >> ibits) != (skmer[i - 1] >> ibits)) ? 1u : 0u;
  }
}

// hscan = exclusive scan of head flags (global).  Group id of sorted element i = hscan[i] + head[i] - 1 (global);
// writes distinct k-mers and local group starts (+ one sentinel per genome), then multiplicities per pv record.
__global__ void groups_kernel(const uint64_t* __restrict__ seg_off, const uint64_t* __restrict__ skmer, uint64_t kmask,
                              const uint32_t* __restrict__ head, const uint32_t* __restrict__ hscan,
                              uint32_t n_genomes, uint32_t* __restrict__ ukmer, uint32_t* __restrict__ ustart, uint32_t ibits) {
  uint32_t g = blockIdx.x;
  uint64_t b = seg_off[g], e = seg_off[g + 1];
  for (uint64_t i = b + (uint64_t)blockIdx.y * blockDim.x + threadIdx.x; i < e; i += (uint64_t)blockDim.x * gridDim.y) {
    if (head[i]) {
      uint32_t gid = hscan[i];
      ukmer[gid] = (uint32_t)((skmer[i] >> ibits) & kmask);
      ustart[gid + g] = (uint32_t)(i - b);
    }
  }
  if (threadIdx.x == 0 && blockIdx.y == 0) {
    // sentinel of genome g sits right after its last group: global group index of next genome's first group
    uint64_t total = seg_off[n_genomes];
    uint32_t next_gid = (e < total) ? hscan[e] : hscan[total - 1] + head[total - 1];  // head[e] is always 1, so hscan[e] = #groups before e; past the end: all groups
    ustart[next_gid + g] = (uint32_t)(e - b);
  }
}

__global__ void mult_kernel(const uint64_t* __restrict__ seg_off, const uint32_t* __restrict__ head,
                            const uint32_t* __restrict__ hscan, const uint32_t* __restrict__ perm,
                            const uint32_t* __restrict__ ustart, uint16_t* __restrict__ pv_mult,
                            const uint64_t* __restrict__ skmer, uint32_t ibits) {
  uint32_t g = blockIdx.x;
  uint64_t b = seg_off[g], e = seg_off[g + 1];
  const uint64_t imask = (1ull << ibits) - 1;
  for (uint64_t i = b + (uint64_t)blockIdx.y * blockDim.x + threadIdx.x; i < e; i += (uint64_t)blockDim.x * gridDim.y) {
    uint32_t gid = hscan[i] + head[i] - 1;
    uint32_t cntv = ustart[gid + g + 1] - ustart[gid + g];
    const uint32_t r = ibits ? (uint32_t)(skmer[i] & imask) : perm[i];
    pv_mult[b + r] = (uint16_t)min(cntv, 65535u);
  }
}

// bucket index over each genome's distinct k-mers: ubucket[g][b] = first index u with (ukmer[u] >> shift) >= b
__global__ void bucket_kernel(const uint64_t* __restrict__ uk_off, const uint32_t* __restrict__ ukmer, uint32_t shift,
                              uint32_t* __restrict__ ubucket) {
  const uint32_t g = blockIdx.x;
  const uint32_t* uk = ukmer + uk_off[g];
  const uint32_t n = (uint32_t)(uk_off[g + 1] - uk_off[g]);
  for (uint32_t b = threadIdx.x; b <= UBUCKETS; b += blockDim.x) {
    uint32_t lo = 0, hi = n;
    while (lo < hi) {
      uint32_t mid = (lo + hi) >> 1;
      if ((uk[mid] >> shift) < b) lo = mid + 1; else hi = mid;
    }
    ubucket[(size_t)g * (UBUCKETS + 1) + b] = lo;
  }
}

// markers: flag distinct values inside each genome's sorted segment
__global__ void marker_head_kernel(const uint64_t* __restrict__ seg_off, const uint64_t* __restrict__ mk,
                                   uint32_t* __restrict__ head) {
  uint32_t g = blockIdx.x;
  uint64_t b = seg_off[g], e = seg_off[g + 1];
  for (uint64_t i = b + (uint64_t)blockIdx.y * blockDim.x + threadIdx.x; i < e; i += (uint64_t)blockDim.x * gridDim.y) head[i] = (i == b || mk[i] != mk[i - 1]) ? 1u : 0u;
}
__global__ void marker_compact_kernel(const uint64_t* __restrict__ mk, const uint32_t* __restrict__ head,
                                      const uint32_t* __restrict__ hscan, uint32_t n, uint64_t mask, uint64_t* __restrict__ out) {
  uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n && head[i]) out[hscan[i]] = mk[i] & mask;
}
__global__ void gather_scan_at_kernel(const uint32_t* __restrict__ scan, const uint64_t* __restrict__ at, uint32_t n,
                                      uint64_t len, uint32_t total, uint64_t* __restrict__ out) {
  uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) out[i] = (at[i] >= len) ? (uint64_t)total : (uint64_t)scan[at[i]];
}

__global__ void gather_scan_at_tail_kernel(const uint32_t* __restrict__ scan, const uint64_t* __restrict__ at, uint32_t n,
                                           uint64_t len, const uint32_t* __restrict__ flag, uint64_t* __restrict__ out) {
  uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) out[i] = (at[i] >= len) ? (uint64_t)(scan[len - 1] + flag[len - 1]) : (uint64_t)scan[at[i]];
}

// ------------------------------------------------------------------------------------------------------------
// host side
// ------------------------------------------------------------------------------------------------------------
// pinned landing space for an asynchronous device->host readback (valid until the next mbox_reset)
static void* mbox_alloc(sk_ctx* ctx, size_t bytes) {
  bytes = (bytes + 63) & ~(size_t)63;
  for (;;) {
    if (ctx->mbox_block < ctx->mbox_blocks.size()) {
      auto& b = ctx->mbox_blocks[ctx->mbox_block];
      if (ctx->mbox_pos + bytes <= b.second) { void* p = b.first + ctx->mbox_pos; ctx->mbox_pos += bytes; return p; }
      ctx->mbox_block++; ctx->mbox_pos = 0;
      continue;
    }
    uint8_t* p = nullptr;
    const size_t cap = std::max<size_t>(bytes, 1u << 20);
    if (cudaHostAlloc((void**)&p, cap, cudaHostAllocPortable) != cudaSuccess) { cudaGetLastError(); return nullptr; }
    ctx->mbox_blocks.push_back({p, cap});
  }
}
void mbox_reset(sk_ctx* ctx) { ctx->mbox_block = 0; ctx->mbox_pos = 0; }

static inline uint32_t div_up(uint64_t a, uint32_t b) { return (uint32_t)((a + b - 1) / b); }

template <typename T>
static int scan_exclusive(sk_ctx* ctx, const T* in, T* out, size_t n) {
  size_t tb = 0;
  SK_CUDA(cub::DeviceScan::ExclusiveSum(nullptr, tb, in, out, n, ctx->stream));
  DTmp<uint8_t> tmp;
  SK_CUDA(tmp.alloc(tb, ctx));
  SK_CUDA(cub::DeviceScan::ExclusiveSum(tmp.p, tb, in, out, n, ctx->stream));
  return SK_OK;
}

void free_set_device(sk_sketch_set* s) {
  void* ptrs[] = {s->pv_kmer, s->pv_pos, s->pv_cc, s->pv_mult, s->kv_pos, s->kv_cc, s->ukmer, s->ustart,
                  s->markers, s->ctg_rec_off, s->d_ctg_len, s->ubucket, s->htab};
  for (void* p : ptrs) if (p) s->ctx->arena.release(p);
  s->pv_kmer = s->pv_pos = s->pv_cc = s->kv_pos = s->kv_cc = s->ukmer = s->ustart = s->ctg_rec_off = s->d_ctg_len = nullptr;
  s->pv_mult = nullptr;
  s->markers = nullptr;
  s->ubucket = nullptr;
  s->htab = nullptr;
}

// per-genome k-mer hash table for the probe kernel: one 8-byte entry holds key, group start and (saturated) group size,
// so a probe costs ~1.2 divergent sector reads instead of a search + two ustart reads
__global__ void hash_build_kernel(const uint64_t* __restrict__ uk_off, const uint64_t* __restrict__ ht_off,
                                  const uint32_t* __restrict__ ukmer, const uint32_t* __restrict__ ustart,
                                  unsigned long long* __restrict__ htab, uint32_t g_base) {
  const uint32_t g = g_base + blockIdx.x;
  const uint64_t cap = ht_off[g + 1] - ht_off[g];
  if (cap == 0) return;
  const uint32_t nb = (uint32_t)(cap >> 2);                              // 4-entry (32-byte) buckets; cap is a power of two >= 16
  const uint32_t bmask = nb - 1;
  const uint32_t shift = 32 - (uint32_t)__ffs((int)nb) + 1;              // 32 - log2(nb)
  const uint32_t* uk = ukmer + uk_off[g];
  const uint32_t* us = ustart + uk_off[g] + g;
  unsigned long long* tab = htab + ht_off[g];
  const uint32_t n = (uint32_t)(uk_off[g + 1] - uk_off[g]);
  for (uint32_t u = blockIdx.y * blockDim.x + threadIdx.x; u < n; u += blockDim.x * gridDim.y) {
    const uint32_t key = uk[u], start = us[u], cntv = us[u + 1] - start;
    // key 0 with start 0 and count 0 cannot occur (count >= 1), so a stored entry is never 0 = "empty"
    const unsigned long long e = ((unsigned long long)key << 32) | ((unsigned long long)start << 12) | (cntv < 4095u ? cntv : 4095u);
    uint32_t b = (key * 0x9E3779B1u) >> shift;
    for (;;) {                      // first free slot of the bucket, front to back; a full bucket spills into the next one
      bool done = false;
#pragma unroll
      for (int sl = 0; sl < 4 && !done; sl++) done = atomicCAS(&tab[4 * b + sl], 0ull, e) == 0ull;
      if (done) break;
      b = (b + 1) & bmask;
    }
  }
}

int build_hash(sk_ctx* ctx, sk_sketch_set* set) {
  cudaStream_t st = ctx->stream;
  const uint32_t G = set->G;
  if (set->htab) { ctx->arena.release(set->htab); set->htab = nullptr; }
  set->ht_off.assign(G + 1, 0);
  const bool force_bucket = getenv("SK_FORCE_BUCKET_PROBE") != nullptr;  // test hook: exercise the large-genome fallback
  for (uint32_t g = 0; g < G && !force_bucket; g++) {
    const uint64_t nuk = set->uk_off[g + 1] - set->uk_off[g], nrec = set->seed_off[g + 1] - set->seed_off[g];
    uint64_t cap = 0;
    if (nuk > 0 && nrec < (1ull << 20)) { cap = 16; while (cap < 2 * nuk) cap <<= 1; }   // start must fit 20 bits
    set->ht_off[g + 1] = set->ht_off[g] + cap;
  }
  const uint64_t total = set->ht_off[G];
  SK_CUDA(ctx->arena.alloc((void**)&set->htab, std::max<uint64_t>(total, 1) * 8));
  // genomes without a table (>= 2^20 records, or the test hook) use the bucket-index search: build that index only then
  bool need_bucket = false;
  for (uint32_t g = 0; g < G; g++) if (set->ht_off[g + 1] == set->ht_off[g] && set->uk_off[g + 1] > set->uk_off[g]) need_bucket = true;
  if (set->ubucket) { ctx->arena.release(set->ubucket); set->ubucket = nullptr; }
  if (need_bucket) {
    DTmp<uint64_t> d_uk2;
    SK_CUDA(d_uk2.alloc(G + 1, ctx));
    SK_CUDA(h2d_small(ctx, d_uk2.p, set->uk_off.data(), (G + 1) * 8));
    SK_CUDA(ctx->arena.alloc((void**)&set->ubucket, (size_t)G * (UBUCKETS + 1) * 4));
    const uint32_t kbits = 2 * set->sp.k;
    const uint32_t shift = kbits > UBUCKET_BITS ? kbits - UBUCKET_BITS : 0;
    bucket_kernel<<<G, 256, 0, st>>>(d_uk2.p, set->ukmer, shift, set->ubucket); count_launch(ctx);
    SK_CUDA(cudaStreamSynchronize(st));
  }
  if (total == 0) return SK_OK;
  SK_CUDA(cudaMemsetAsync(set->htab, 0, total * 8, st));
  DTmp<uint64_t> d_uk, d_ht;
  SK_CUDA(d_uk.alloc(G + 1, ctx)); SK_CUDA(d_ht.alloc(G + 1, ctx));
  SK_CUDA(h2d_small(ctx, d_uk.p, set->uk_off.data(), (G + 1) * 8));
  SK_CUDA(h2d_small(ctx, d_ht.p, set->ht_off.data(), (G + 1) * 8));
  hash_build_kernel<<<dim3(G, 32), 256, 0, st>>>(d_uk.p, d_ht.p, set->ukmer, set->ustart, set->htab, 0); count_launch(ctx);
  SK_CUDA(cudaStreamSynchronize(st));
  return SK_OK;
}

// Tables of the genomes [g_begin, G) of a set whose earlier genomes already have theirs (in-place growth): the new
// tables are appended to set->htab (grown if its capacity is exceeded).  Falls back to the full rebuild when a new genome
// is too large for a table (needs the bucket index).
int build_hash_range(sk_ctx* ctx, sk_sketch_set* set, uint32_t g_begin) {
  cudaStream_t st = ctx->stream;
  const uint32_t G = set->G;
  if (set->ht_off.size() != (size_t)g_begin + 1 || set->ubucket || getenv("SK_FORCE_BUCKET_PROBE")) { set->capHT = 0; return build_hash(ctx, set); }
  std::vector<uint64_t> ht(set->ht_off);
  for (uint32_t g = g_begin; g < G; g++) {
    const uint64_t nuk = set->uk_off[g + 1] - set->uk_off[g], nrec = set->seed_off[g + 1] - set->seed_off[g];
    uint64_t cap = 0;
    if (nuk > 0) {
      if (nrec >= (1ull << 20)) { set->capHT = 0; return build_hash(ctx, set); }
      cap = 16; while (cap < 2 * nuk) cap <<= 1;
    }
    ht.push_back(ht.back() + cap);
  }
  const uint64_t old_total = ht[g_begin], total = ht[G];
  const size_t have = set->capHT ? set->capHT : std::max<uint64_t>(old_total, 1);
  if (total > have) {
    const size_t ncap = std::max<size_t>(total, have + have / 2);
    unsigned long long* nt = nullptr;
    SK_CUDA(ctx->arena.alloc((void**)&nt, ncap * 8));
    if (old_total) SK_CUDA(cudaMemcpyAsync(nt, set->htab, old_total * 8, cudaMemcpyDeviceToDevice, st));
    SK_CUDA(cudaStreamSynchronize(st));
    ctx->arena.release(set->htab);
    set->htab = nt; set->capHT = ncap;
  }
  set->ht_off = ht;
  if (total == old_total) return SK_OK;
  SK_CUDA(cudaMemsetAsync(set->htab + old_total, 0, (total - old_total) * 8, st));
  DTmp<uint64_t> d_uk, d_ht;
  SK_CUDA(d_uk.alloc(G + 1, ctx)); SK_CUDA(d_ht.alloc(G + 1, ctx));
  SK_CUDA(h2d_small(ctx, d_uk.p, set->uk_off.data(), (G + 1) * 8));
  SK_CUDA(h2d_small(ctx, d_ht.p, set->ht_off.data(), (G + 1) * 8));
  hash_build_kernel<<<dim3(G - g_begin, 32), 256, 0, st>>>(d_uk.p, d_ht.p, set->ukmer, set->ustart, set->htab, g_begin); count_launch(ctx);
  SK_CUDA(cudaStreamSynchronize(st));
  return SK_OK;
}

// Given the position view (pv_kmer/pv_pos/pv_cc filled, set->seed_off known) and the raw (unsorted, possibly
// duplicated) markers per genome, build the k-mer view, groups, multiplicities and the sorted distinct marker arrays.
int build_views(sk_ctx* ctx, sk_sketch_set* set, uint64_t* d_marker_raw, const uint64_t* raw_mk_off) {
  // Host synchronisations: ONE in the middle (the raw marker counts are needed to size the marker sort; by then the whole
  // k-mer view is queued behind it, so the device does not idle) and one at the end.  Everything whose size only the device
  // knows yet (distinct k-mers, distinct markers) is allocated at its upper bound and the totals are read back at the end.
  const uint32_t G = set->G;
  const size_t S = set->S;
  cudaStream_t st = ctx->stream;
  DTmp<uint64_t> d_seed_off, d_rawmk_off;
  SK_CUDA(d_seed_off.alloc(G + 1, ctx));
  SK_CUDA(h2d_small(ctx, d_seed_off.p, set->seed_off.data(), (G + 1) * 8));
  SK_CUDA(ctx->arena.alloc((void**)&set->kv_pos, std::max<size_t>(S, 1) * 4));
  SK_CUDA(ctx->arena.alloc((void**)&set->kv_cc, std::max<size_t>(S, 1) * 4));
  SK_CUDA(ctx->arena.alloc((void**)&set->pv_mult, std::max<size_t>(S, 1) * 2));
  set->uk_off.assign(G + 1, 0);
  uint64_t* h_ukoff = (uint64_t*)mbox_alloc(ctx, (size_t)(G + 1) * 8);
  uint64_t* h_mkoff = (uint64_t*)mbox_alloc(ctx, (size_t)(G + 1) * 8);
  if (!h_ukoff || !h_mkoff) { ctx->err = "out of pinned host memory"; return SK_ERR_NOMEM; }
  if (S > 0) {
    if (S >= (1ull << 31)) { ctx->err = "sub-batch has >= 2^31 seed records"; return SK_ERR_PARAM; }
    DTmp<uint32_t> vals, perm, head, hscan;
    DTmp<uint64_t> keys, skmer;
    SK_CUDA(keys.alloc(S, ctx)); SK_CUDA(skmer.alloc(S, ctx));
    SK_CUDA(head.alloc(S + 1, ctx)); SK_CUDA(hscan.alloc(S + 1, ctx));
    const uint32_t kbits = std::min(32u, 2 * set->sp.k);
    const uint32_t gbits = G > 1 ? 32 - (uint32_t)__builtin_clz(G - 1) : 0;     // bits of a genome index 0 .. G-1
    const uint64_t kmask = (kbits >= 64) ? ~0ull : ((1ull << kbits) - 1);
    uint64_t max_rec = 1;
    for (uint32_t g = 0; g < G; g++) max_rec = std::max<uint64_t>(max_rec, set->seed_off[g + 1] - set->seed_off[g]);
    uint32_t ibits = max_rec > 1 ? 64 - (uint32_t)__builtin_clzll(max_rec - 1) : 1;   // bits of a record index inside its genome
    if (ibits + kbits + gbits > 64 || getenv("SK_KVIEW_SORT_PAIRS")) ibits = 0;                // does not fit: (key, index) pairs
    if (!ibits) { SK_CUDA(vals.alloc(S, ctx)); SK_CUDA(perm.alloc(S, ctx)); }
    kview_keys_kernel<<<dim3(G, 8), 256, 0, st>>>(d_seed_off.p, set->pv_kmer, kbits, ibits, keys.p, vals.p); count_launch(ctx);
    size_t tb = 0;
    DTmp<uint8_t> tmp;
    if (ibits) {
      SK_CUDA(cub::DeviceRadixSort::SortKeys(nullptr, tb, keys.p, skmer.p, (int)S, (int)ibits, (int)(ibits + kbits + gbits), st));
      SK_CUDA(tmp.alloc(tb, ctx));
      SK_CUDA(cub::DeviceRadixSort::SortKeys(tmp.p, tb, keys.p, skmer.p, (int)S, (int)ibits, (int)(ibits + kbits + gbits), st));
    } else {
      SK_CUDA(cub::DeviceRadixSort::SortPairs(nullptr, tb, keys.p, skmer.p, vals.p, perm.p, (int)S, 0, (int)(kbits + gbits), st));
      SK_CUDA(tmp.alloc(tb, ctx));
      SK_CUDA(cub::DeviceRadixSort::SortPairs(tmp.p, tb, keys.p, skmer.p, vals.p, perm.p, (int)S, 0, (int)(kbits + gbits), st));
    }
    count_launch(ctx);
    kview_gather_kernel<<<dim3(G, 8), 256, 0, st>>>(d_seed_off.p, skmer.p, perm.p, set->pv_pos, set->pv_cc, set->kv_pos,
                                           set->kv_cc, head.p, ibits); count_launch(ctx);
    SK_TRY(scan_exclusive<uint32_t>(ctx, head.p, hscan.p, S));
    // per-genome group offsets (+ the total in the last slot) -> host, asynchronously
    DTmp<uint64_t> d_ukoff;
    SK_CUDA(d_ukoff.alloc(G + 1, ctx));
    gather_scan_at_tail_kernel<<<div_up(G + 1, 256), 256, 0, st>>>(hscan.p, d_seed_off.p, G + 1, S, head.p, d_ukoff.p); count_launch(ctx);
    SK_CUDA(cudaMemcpyAsync(h_ukoff, d_ukoff.p, (size_t)(G + 1) * 8, cudaMemcpyDeviceToHost, st));
    SK_CUDA(ctx->arena.alloc((void**)&set->ukmer, S * 4));                       // upper bound: distinct k-mers <= records
    SK_CUDA(ctx->arena.alloc((void**)&set->ustart, (size_t)(S + G + 1) * 4));
    groups_kernel<<<dim3(G, 8), 256, 0, st>>>(d_seed_off.p, skmer.p, kmask, head.p, hscan.p, G, set->ukmer, set->ustart, ibits); count_launch(ctx);
    mult_kernel<<<dim3(G, 8), 256, 0, st>>>(d_seed_off.p, head.p, hscan.p, perm.p, set->ustart, set->pv_mult, skmer.p, ibits); count_launch(ctx);
  } else {
    set->U = 0;
    SK_CUDA(ctx->arena.alloc((void**)&set->ukmer, 4));
    SK_CUDA(ctx->arena.alloc((void**)&set->ustart, (size_t)(G + 1) * 4));
    SK_CUDA(cudaMemsetAsync(set->ustart, 0, (size_t)(G + 1) * 4, st));
    for (uint32_t g = 0; g <= G; g++) h_ukoff[g] = 0;
  }
  SK_CUDA(cudaStreamSynchronize(st));      // raw marker offsets (queued by the caller) and group offsets have landed
  for (uint32_t g = 0; g <= G; g++) set->uk_off[g] = h_ukoff[g];
  set->U = (size_t)set->uk_off[G];
  // ---- markers: per-genome sort + dedup (HashSet semantics, reference src/types.rs:269)
  const size_t MR = raw_mk_off[G];
  set->mk_off.assign(G + 1, 0);
  if (MR > 0) {
    if (MR >= (1ull << 31)) { ctx->err = "sub-batch has >= 2^31 markers"; return SK_ERR_PARAM; }
    SK_CUDA(d_rawmk_off.alloc(G + 1, ctx));
    SK_CUDA(h2d_small(ctx, d_rawmk_off.p, raw_mk_off, (G + 1) * 8));
    DTmp<uint64_t> sorted;
    SK_CUDA(sorted.alloc(MR, ctx));
    size_t tb = 0;
    const uint32_t mgbits = G > 1 ? 32 - (uint32_t)__builtin_clz(G - 1) : 0;
    const bool global_sort = 2 * MARKER_K + mgbits <= 64;      // one device-wide sort of (genome << 42 | marker); else per-genome segments
    DTmp<uint8_t> tmp;
    if (global_sort) {
      marker_keys_kernel<<<dim3(G, 8), 256, 0, st>>>(d_rawmk_off.p, d_marker_raw); count_launch(ctx);
      SK_CUDA(cub::DeviceRadixSort::SortKeys(nullptr, tb, d_marker_raw, sorted.p, (int)MR, 0, (int)(2 * MARKER_K + mgbits), st));
      SK_CUDA(tmp.alloc(tb, ctx));
      SK_CUDA(cub::DeviceRadixSort::SortKeys(tmp.p, tb, d_marker_raw, sorted.p, (int)MR, 0, (int)(2 * MARKER_K + mgbits), st));
    } else {
      SK_CUDA(cub::DeviceSegmentedRadixSort::SortKeys(nullptr, tb, d_marker_raw, sorted.p, (int)MR, (int)G, d_rawmk_off.p,
                                                      d_rawmk_off.p + 1, 0, 2 * MARKER_K, st));
      SK_CUDA(tmp.alloc(tb, ctx));
      SK_CUDA(cub::DeviceSegmentedRadixSort::SortKeys(tmp.p, tb, d_marker_raw, sorted.p, (int)MR, (int)G, d_rawmk_off.p,
                                                      d_rawmk_off.p + 1, 0, 2 * MARKER_K, st));
    }
    count_launch(ctx);
    DTmp<uint32_t> head, hscan;
    SK_CUDA(head.alloc(MR, ctx)); SK_CUDA(hscan.alloc(MR, ctx));
    marker_head_kernel<<<dim3(G, 8), 256, 0, st>>>(d_rawmk_off.p, sorted.p, head.p); count_launch(ctx);
    SK_TRY(scan_exclusive<uint32_t>(ctx, head.p, hscan.p, MR));
    SK_CUDA(ctx->arena.alloc((void**)&set->markers, MR * 8));                 // upper bound: distinct markers <= raw markers
    marker_compact_kernel<<<div_up(MR, 256), 256, 0, st>>>(sorted.p, head.p, hscan.p, (uint32_t)MR, global_sort ? ((1ull << (2 * MARKER_K)) - 1) : ~0ull, set->markers); count_launch(ctx);
    DTmp<uint64_t> d_mkoff;
    SK_CUDA(d_mkoff.alloc(G + 1, ctx));
    gather_scan_at_tail_kernel<<<div_up(G + 1, 256), 256, 0, st>>>(hscan.p, d_rawmk_off.p, G + 1, MR, head.p, d_mkoff.p); count_launch(ctx);
    SK_CUDA(cudaMemcpyAsync(h_mkoff, d_mkoff.p, (size_t)(G + 1) * 8, cudaMemcpyDeviceToHost, st));
    SK_CUDA(cudaStreamSynchronize(st));
    for (uint32_t g = 0; g <= G; g++) set->mk_off[g] = h_mkoff[g];
    set->M = (size_t)set->mk_off[G];
  } else {
    set->M = 0;
    SK_CUDA(ctx->arena.alloc((void**)&set->markers, 8));
  }
  return SK_OK;
}

struct PopcOp { using result_type = uint32_t; __device__ __forceinline__ uint32_t operator()(uint32_t m) const { return (uint32_t)__popc(m); } };

// Seeds all contigs of one sub-batch.  The sequence arrives either as ASCII resident on the device (contig i at
// src.d_ascii + contig_off[i] - src.ascii_base; converted by pack_kernel) or, for the first src.n_packed contigs, already
// as 2-bit units + N mask inside src.d_P / src.d_NM (packed on the host, api.cu, or handed over by sk_sketch_batch_2bit).
// Unit layout: contig i owns units [cuoff[i], cuoff[i+1]), cuoff = prefix sum of ceil(len / 32).
int sketch_batch_device(sk_ctx* ctx, const SeedSrc& src, const uint64_t* contig_off, uint32_t n_contigs,
                        const uint32_t* genome_of_contig, uint32_t n_genomes, const sk_sketch_params* sp, sk_sketch_set** out) {
  cudaStream_t st = ctx->stream;
  const uint32_t G = n_genomes;
  sk_sketch_set* set = new sk_sketch_set();
  set->ctx = ctx; set->sp = *sp; set->G = G;
  struct Guard { sk_sketch_set* s; ~Guard() { if (s) { free_set_device(s); delete s; } } } guard{set};

  // ---- host-side layout
  std::vector<uint64_t> coff(n_contigs + 1);
  std::vector<uint32_t> cuoff(n_contigs + 1), clen(n_contigs), clocal(n_contigs);
  set->ctg_off.assign(G + 1, 0);
  set->total_len.assign(G, 0);
  set->ctg_len.resize(n_contigs);
  uint64_t units = 0;
  uint32_t prev_g = 0, rank = 0;
  for (uint32_t i = 0; i < n_contigs; i++) {
    uint64_t len = contig_off[i + 1] - contig_off[i];
    if (contig_off[i + 1] < contig_off[i] || len >= (1ull << 32) - 65536) { ctx->err = "contig length out of range (u32 positions, src/types.rs:52; pos + 20000 must not wrap, src/chain.rs:743)"; return SK_ERR_PARAM; }
    uint32_t g = genome_of_contig[i];
    if (g >= G || g < prev_g) { ctx->err = "genome_of_contig must be non-decreasing and < n_genomes"; return SK_ERR_PARAM; }
    if (g != prev_g || i == 0) rank = 0;
    prev_g = g;
    if (rank >= (1u << 30)) { ctx->err = "contig index exceeds 30 bits (src/types.rs:136)"; return SK_ERR_PARAM; }
    coff[i] = contig_off[i] - src.ascii_base;
    cuoff[i] = (uint32_t)units;
    clen[i] = (uint32_t)len;
    clocal[i] = rank++;
    set->ctg_len[i] = (uint32_t)len;
    set->ctg_off[g + 1]++;
    set->total_len[g] += len;
    units += (len + 31) / 32;
    if (units >= (1ull << 31)) { ctx->err = "sub-batch too large (>= 2^31 units)"; return SK_ERR_PARAM; }
  }
  coff[n_contigs] = contig_off[n_contigs] - src.ascii_base;
  cuoff[n_contigs] = (uint32_t)units;
  for (uint32_t g = 0; g < G; g++) set->ctg_off[g + 1] += set->ctg_off[g];
  set->C = n_contigs;
  set->name_rank.resize(G);
  for (uint32_t g = 0; g < G; g++) set->name_rank[g] = g;
  const uint32_t NU = (uint32_t)units;
  const uint32_t n_packed = std::min(src.n_packed, n_contigs);
  if (n_packed && (!src.d_P || !src.d_NM)) { ctx->err = "packed contigs without unit arrays"; return SK_ERR_PARAM; }
  // coarse unit -> contig index: contig of every 256th unit (= the last contig starting at or before it)
  std::vector<uint32_t> ucoarse(((size_t)NU >> UCOARSE_SHIFT) + 2, n_contigs ? n_contigs - 1 : 0);
  {
    uint32_t ci = 0;
    for (size_t j = 0; ((uint64_t)j << UCOARSE_SHIFT) < NU; j++) {
      const uint32_t u = (uint32_t)(j << UCOARSE_SHIFT);
      while (ci + 1 < n_contigs && cuoff[ci + 1] <= u) ci++;
      ucoarse[j] = ci;
    }
  }

  SK_CUDA(ctx->arena.alloc((void**)&set->d_ctg_len, std::max<size_t>(n_contigs, 1) * 4));
  SK_CUDA(ctx->arena.alloc((void**)&set->ctg_rec_off, (size_t)(n_contigs + G + 1) * 4));
  set->seed_off.assign(G + 1, 0);

  DTmp<uint64_t> d_coff, Pown;
  DTmp<uint32_t> d_cuoff, d_clen, d_clocal, d_ucoarse, NMown, PM, uoff;
  mbox_reset(ctx);                           // no readback of an earlier sub-batch is in flight (each one ends synchronised)
  uint64_t* h_raw_mk_off = (uint64_t*)mbox_alloc(ctx, (size_t)(G + 1) * 8);    // raw markers per genome (prefix offsets), pinned
  if (h_raw_mk_off) for (uint32_t g = 0; g <= G; g++) h_raw_mk_off[g] = 0;
  DTmp<uint64_t> mkv, mraw;
  if (NU > 0) {
    SK_CUDA(d_coff.alloc(n_contigs + 1, ctx)); SK_CUDA(d_cuoff.alloc(n_contigs + 1, ctx));
    SK_CUDA(d_clen.alloc(n_contigs, ctx)); SK_CUDA(d_clocal.alloc(n_contigs, ctx)); SK_CUDA(d_ucoarse.alloc(ucoarse.size(), ctx));
    SK_CUDA(h2d_small(ctx, d_coff.p, coff.data(), (n_contigs + 1) * 8));
    SK_CUDA(h2d_small(ctx, d_cuoff.p, cuoff.data(), (n_contigs + 1) * 4));
    SK_CUDA(h2d_small(ctx, d_clen.p, clen.data(), n_contigs * 4));
    SK_CUDA(h2d_small(ctx, d_clocal.p, clocal.data(), n_contigs * 4));
    SK_CUDA(h2d_small(ctx, d_ucoarse.p, ucoarse.data(), ucoarse.size() * 4));
    SK_CUDA(h2d_small(ctx, set->d_ctg_len, clen.data(), n_contigs * 4));
    uint64_t* P = src.d_P; uint32_t* NM = src.d_NM;
    if (!P) { SK_CUDA(Pown.alloc(NU, ctx)); SK_CUDA(NMown.alloc(NU, ctx)); P = Pown.p; NM = NMown.p; }
    SK_CUDA(PM.alloc(NU, ctx)); SK_CUDA(uoff.alloc(NU, ctx));

    const uint32_t u_ascii = cuoff[n_packed];            // first unit that still has to be converted on the device
    if (u_ascii < NU) {
      if (!src.d_ascii) { ctx->err = "ASCII contigs without a device buffer"; return SK_ERR_PARAM; }
      SK_LAUNCH(ctx, "pack_kernel", (pack_kernel<<<div_up(NU - u_ascii, PACK_THREADS), PACK_THREADS, 0, st>>>(
          src.d_ascii, d_coff.p, d_cuoff.p, d_clen.p, d_ucoarse.p, u_ascii, NU, P, NM, ctx->seed_scalar ? 1 : 0)));
    }
    const uint64_t seed_mask = ~0ull >> (64 - 2 * sp->k);
    const uint64_t thr = ~0ull / sp->c, thr_m = ~0ull / sp->marker_c;  // src/avx2_seeding.rs:93-94
    {
      const uint32_t scalar_k = ctx->seed_scalar ? sp->k : 0;     // scalar fmh_seeds semantics (sk_ctx_set_seeding_semantics)
      const int hv = (getenv("SK_HASHPASS_VARIANT") && !scalar_k) ? atoi(getenv("SK_HASHPASS_VARIANT")) : 0;
      const uint32_t c24 = 1u << 8, c14 = 1u << 18, c28 = 1u << 4;     // 2^(32 - s) for the xor-shift distances 24 / 14 / 28
      const uint32_t grid = div_up(NU, HASH_THREADS);
      if (hv == 1) SK_LAUNCH(ctx, "hashpass_kernel", (hashpass_kernel<1><<<grid, HASH_THREADS, 0, st>>>(P, NM, d_ucoarse.p, d_cuoff.p, d_clen.p, NU, seed_mask, thr, PM.p, c24, c14, c28, scalar_k)));
      else if (hv == 2) SK_LAUNCH(ctx, "hashpass_kernel", (hashpass_kernel<2><<<grid, HASH_THREADS, 0, st>>>(P, NM, d_ucoarse.p, d_cuoff.p, d_clen.p, NU, seed_mask, thr, PM.p, c24, c14, c28, scalar_k)));
      else SK_LAUNCH(ctx, "hashpass_kernel", (hashpass_kernel<0><<<grid, HASH_THREADS, 0, st>>>(P, NM, d_ucoarse.p, d_cuoff.p, d_clen.p, NU, seed_mask, thr, PM.p, c24, c14, c28, scalar_k)));
    }
    {   // record offset of every unit = exclusive scan of the pass-mask popcounts (no separate count array)
      auto cnt_it = thrust::make_transform_iterator((const uint32_t*)PM.p, PopcOp());
      size_t tb = 0;
      SK_CUDA(cub::DeviceScan::ExclusiveSum(nullptr, tb, cnt_it, uoff.p, (int)NU, st));
      DTmp<uint8_t> tmp;
      SK_CUDA(tmp.alloc(tb, ctx));
      SK_CUDA(cub::DeviceScan::ExclusiveSum(tmp.p, tb, cnt_it, uoff.p, (int)NU, st));
      count_launch(ctx, 2);
    }
    // record offset of every contig's first unit (-> per-genome offsets and per-contig record offsets); the entry past the last
    // contig is the total number of records, computed on the device: ONE host synchronisation delivers everything the host
    // needs to size the record arrays and lay out the set
    DTmp<uint32_t> d_crec;
    SK_CUDA(d_crec.alloc(n_contigs + 1, ctx));
    gather_u32_tail_kernel<<<div_up(n_contigs + 1, 256), 256, 0, st>>>(uoff.p, d_cuoff.p, n_contigs + 1, NU, PM.p, 1, d_crec.p); count_launch(ctx);
    uint32_t* crec = (uint32_t*)mbox_alloc(ctx, (size_t)(n_contigs + 1) * 4);
    if (!crec || !h_raw_mk_off) { ctx->err = "out of pinned host memory"; return SK_ERR_NOMEM; }
    SK_CUDA(cudaMemcpyAsync(crec, d_crec.p, (size_t)(n_contigs + 1) * 4, cudaMemcpyDeviceToHost, st));
    SK_CUDA(cudaStreamSynchronize(st));
    const uint32_t S = crec[n_contigs];      // cuoff[n_contigs] == NU: "past the end"
    set->S = S;
    SK_CUDA(ctx->arena.alloc((void**)&set->pv_kmer, std::max<size_t>(S, 1) * 4));
    SK_CUDA(ctx->arena.alloc((void**)&set->pv_pos, std::max<size_t>(S, 1) * 4));
    SK_CUDA(ctx->arena.alloc((void**)&set->pv_cc, std::max<size_t>(S, 1) * 4));
    SK_CUDA(mkv.alloc(S, ctx));
    SK_LAUNCH(ctx, "expand_kernel", (expand_kernel<<<div_up(NU, 256), 256, 0, st>>>(
        P, d_ucoarse.p, d_cuoff.p, d_clocal.p, NU, PM.p, uoff.p, seed_mask, thr_m, set->pv_kmer, set->pv_pos, set->pv_cc, mkv.p)));
    // per-genome record offsets + per-contig local record offsets (with one sentinel per genome)
    std::vector<uint32_t> crl(n_contigs + G + 1, 0);
    for (uint32_t g = 0; g < G; g++) {
      uint64_t c0 = set->ctg_off[g], c1 = set->ctg_off[g + 1];
      uint32_t base = (c0 < n_contigs) ? crec[c0] : S;
      set->seed_off[g] = base;
      for (uint64_t c = c0; c < c1; c++) crl[c + g] = crec[c] - base;
      uint32_t endrec = (c1 < n_contigs) ? crec[c1] : S;
      crl[c1 + g] = endrec - base;
    }
    set->seed_off[G] = S;
    SK_CUDA(h2d_small(ctx, set->ctg_rec_off, crl.data(), (size_t)(n_contigs + G) * 4));
    // raw markers: compact the flagged values (order inside a genome is irrelevant: they are sorted + deduped next).  Their
    // number is not known to the host yet: the buffer takes the upper bound (one per record), the per-genome offsets travel to
    // the host asynchronously and are read after build_views' first synchronisation.
    if (S > 0) {
      DTmp<uint32_t> mflag, mscan;
      SK_CUDA(mflag.alloc(S, ctx)); SK_CUDA(mscan.alloc(S, ctx));
      marker_flag_kernel<<<div_up(S, 256), 256, 0, st>>>(mkv.p, S, mflag.p); count_launch(ctx);
      SK_TRY(scan_exclusive<uint32_t>(ctx, mflag.p, mscan.p, S));
      DTmp<uint64_t> d_so, d_mo;
      SK_CUDA(d_so.alloc(G + 1, ctx)); SK_CUDA(d_mo.alloc(G + 1, ctx));
      SK_CUDA(h2d_small(ctx, d_so.p, set->seed_off.data(), (G + 1) * 8));
      SK_CUDA(mraw.alloc(S, ctx));
      marker_scatter_kernel<<<div_up(S, 256), 256, 0, st>>>(mkv.p, mscan.p, S, mraw.p); count_launch(ctx);
      gather_scan_at_tail_kernel<<<div_up(G + 1, 256), 256, 0, st>>>(mscan.p, d_so.p, G + 1, S, mflag.p, d_mo.p); count_launch(ctx);
      SK_CUDA(cudaMemcpyAsync(h_raw_mk_off, d_mo.p, (size_t)(G + 1) * 8, cudaMemcpyDeviceToHost, st));
    }
  } else {
    set->S = 0;
    SK_CUDA(ctx->arena.alloc((void**)&set->pv_kmer, 4)); SK_CUDA(ctx->arena.alloc((void**)&set->pv_pos, 4)); SK_CUDA(ctx->arena.alloc((void**)&set->pv_cc, 4));
    SK_CUDA(cudaMemsetAsync(set->ctg_rec_off, 0, (size_t)(n_contigs + G + 1) * 4, st));
  }
  // free the big per-base temporaries before the sort temporaries are allocated
  Pown.release(); NMown.release(); PM.release(); uoff.release(); mkv.release();
  if (!h_raw_mk_off) { ctx->err = "out of pinned host memory"; return SK_ERR_NOMEM; }
  SK_TRY(build_views(ctx, set, mraw.p, h_raw_mk_off));
  SK_CUDA(cudaStreamSynchronize(st));
  guard.s = nullptr;
  *out = set;
  return SK_OK;
}

}  // namespace sk
