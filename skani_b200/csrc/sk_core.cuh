// sk_core.cuh -- per-item arithmetic of the hot path as __host__ __device__ inline functions.
// Included by the CUDA kernels (device) and by tests/emu (host, g++) so the bit-level logic can be
// checked against the oracle without a GPU.  No CPU product path uses these: the library entry points
// only ever launch kernels.
#pragma once
#include <stdint.h>

#if defined(__CUDACC__)
#define SK_HD __host__ __device__ __forceinline__
#else
#define SK_HD inline
#endif

namespace sk {

constexpr int MARKER_K = 21;             // K_MARKER_DNA, reference src/params.rs:35
constexpr uint32_t UNIT_BASES = 32;      // one packed unit = 32 bases = one u64 of 2-bit codes + one u32 N-mask

// Thomas Wang 64-bit mix, reference src/types.rs:86-96 (mm_hash64) / src/avx2_seeding.rs:7-30 (mm_hash256)
SK_HD uint64_t mm_hash64(uint64_t key) {
  key = ~(key + (key << 21));
  key = key ^ (key >> 24);
  key = key * 265;  // (key + (key << 3)) + (key << 8)
  key = key ^ (key >> 14);
  key = key * 21;   // (key + (key << 2)) + (key << 4)
  key = key ^ (key >> 28);
  key = key + (key << 31);
  return key;
}

// ASCII -> (2-bit code | isN << 2), reference src/types.rs:40-49 (BYTE_TO_SEQ) + the 'N' (78) test of
// src/avx2_seeding.rs:115-126.  Lower-case n and IUPAC codes are plain 'A' on the AVX2 path.
SK_HD uint32_t ascii_code(uint32_t b) {
  uint32_t u = b & 0xDFu;  // fold case for letters
  uint32_t v = 0;
  if (u == 'C') v = 1;
  else if (u == 'G') v = 2;
  else if (u == 'T' || u == 'U') v = 3;
  if (b < 4) v = b;        // table rows 0..3 map to themselves
  if ((b & 0xC0u) != 0x40u && b >= 4) v = 0;  // only 0x40..0x7F are letters (guards e.g. 0x03|0x20 style aliases)
  if (b == 78) v |= 4;
  return v;
}

// Four ASCII bytes -> four 2-bit codes (bits 2i..2i+1 = byte i) + four 'N' flags, SIMD-in-register.
// Letters ACGTU in either case: code = ((b >> 1) ^ (b >> 2)) & 3 (A 0, C 1, G 2, T/U 3 = BYTE_TO_SEQ, src/types.rs:40-49).
// The word takes the arithmetic path only if all four bytes are such letters (checked by rebuilding the expected
// upper-case byte from the code); anything else (N, IUPAC, table rows 0..3, padding) goes through ascii_code per byte.
SK_HD void pack_word(uint32_t x, uint32_t& code8, uint32_t& n4, bool small_n = false) {
  const uint32_t t = ((x >> 1) ^ (x >> 2)) & 0x03030303u;
  const uint32_t lo = t & 0x01010101u, hi = (t >> 1) & 0x01010101u, lh = lo & hi;
  const uint32_t expect = 0x41414141u + 2u * lo + 6u * hi + 11u * lh;     // 'A' 'C' 'G' 'T' per byte (no carries: max 0x54)
  const uint32_t u = x & 0xDFDFDFDFu;                                     // fold case
  // (the scalar seeder also treats 'n' as a break, src/seeding.rs:273: with small_n the N-mask flags it; 'n' is never a valid letter)
  if ((((u ^ expect) & ~lh)) == 0u) {                                     // T/U differ in bit 0 only
    code8 = (t * 0x00041041u) >> 18 & 0xFFu;                              // gather the four 2-bit fields (disjoint partial products)
    n4 = 0;
    return;
  }
  uint32_t c = 0, n = 0;
#pragma unroll
  for (int b = 0; b < 4; b++) {
    const uint32_t byte = (x >> (8 * b)) & 0xFFu;
    const uint32_t v = ascii_code(byte);
    c |= (v & 3u) << (2 * b);
    n |= ((v >> 2) | ((small_n && byte == 110u) ? 1u : 0u)) << b;
  }
  code8 = c; n4 = n;
}

// reverse the order of the 32 2-bit fields of a u64 (base j <-> base 31-j)
SK_HD uint64_t pair_reverse64(uint64_t x) {
  x = ((x >> 2) & 0x3333333333333333ull) | ((x & 0x3333333333333333ull) << 2);
  x = ((x >> 4) & 0x0F0F0F0F0F0F0F0Full) | ((x & 0x0F0F0F0F0F0F0F0Full) << 4);
  x = ((x >> 8) & 0x00FF00FF00FF00FFull) | ((x & 0x00FF00FF00FF00FFull) << 8);
  x = ((x >> 16) & 0x0000FFFF0000FFFFull) | ((x & 0x0000FFFF0000FFFFull) << 16);
  x = (x >> 32) | (x << 32);
  return x;
}

// 64 bits of the 128-bit value (hi:lo) starting at bit `sh` (0 <= sh < 128); bits beyond 127 read as 0
SK_HD uint64_t extract128(uint64_t lo, uint64_t hi, uint32_t sh) {
  if (sh == 0) return lo;
  if (sh < 64) return (lo >> sh) | (hi << (64 - sh));
  if (sh == 64) return hi;
  return hi >> (sh - 64);
}

// Window arithmetic.  `lo` = packed unit u-1 (0 for the first unit of a contig), `hi` = packed unit u; window j
// (0..31) ends at base 32*ul + j.  Packed layout: base b of a unit in bits [2b, 2b+1].
// Forward 21-mer F21 has the newest base in its low bits (reference src/seeding.rs:278-280) = pair-reversed stream;
// reverse 21-mer R21 has the complement of the OLDEST base in its low bits (src/seeding.rs:281-283) = complemented stream.
struct WindowCtx {
  uint64_t c_lo, c_hi;  // complemented little-endian stream (~lo, ~hi): R21(j) = extract(c, 24 + 2j) & M42
  uint64_t t_lo, t_hi;  // pair-reversed stream: t = pairrev(hi:lo) => t_lo = pairrev(hi), t_hi = pairrev(lo); F21(j) = extract(t, 62 - 2j) & M42
};
SK_HD WindowCtx make_window_ctx(uint64_t lo, uint64_t hi) {
  WindowCtx w;
  w.c_lo = ~lo; w.c_hi = ~hi;
  w.t_lo = pair_reverse64(hi); w.t_hi = pair_reverse64(lo);
  return w;
}
SK_HD uint64_t window_f21(const WindowCtx& w, uint32_t j) { return extract128(w.t_lo, w.t_hi, 62 - 2 * j) & ((1ull << 42) - 1); }
SK_HD uint64_t window_r21(const WindowCtx& w, uint32_t j) { return extract128(w.c_lo, w.c_hi, 24 + 2 * j) & ((1ull << 42) - 1); }

// Seed of window j: Fs = low 2k bits of F21 (last k bases), Rs = low 2k bits of R21 (revcomp of the FIRST k bases),
// canonical = Fs < Rs, seed = canonical ? Fs : Rs (src/avx2_seeding.rs:145-150; tie -> Rs, same value).
SK_HD uint32_t window_seed(const WindowCtx& w, uint32_t j, uint64_t seed_mask, bool* canonical) {
  uint64_t fs = window_f21(w, j) & seed_mask;
  uint64_t rs = window_r21(w, j) & seed_mask;
  *canonical = fs < rs;
  return (uint32_t)(fs < rs ? fs : rs);
}
SK_HD uint64_t window_marker(const WindowCtx& w, uint32_t j) {  // min(F21, R21), src/avx2_seeding.rs:148,188-194
  uint64_t f = window_f21(w, j), r = window_r21(w, j);
  return r > f ? f : r;
}

// Which windows of unit `ul` of a contig of length n exist at all: ends e = 32*ul + j with 20 <= e < 4q + 20,
// q = (n - 20) / 4 (src/avx2_seeding.rs:48-52,108: the last (n-20) mod 4 windows are never examined); n < 42 -> none (:56-58).
SK_HD uint32_t unit_valid_mask(uint32_t n, uint32_t ul) {
  if (n < 2 * MARKER_K) return 0;
  uint32_t q = (n - 20) / 4;
  uint64_t e_lo = 20, e_hi = 4ull * q + 20;  // [e_lo, e_hi)
  uint64_t b = 32ull * ul;
  uint32_t m = 0xFFFFFFFFu;
  if (b + 32 <= e_lo || b >= e_hi) return 0;
  if (b < e_lo) m &= 0xFFFFFFFFu << (uint32_t)(e_lo - b);
  if (b + 32 > e_hi) m &= 0xFFFFFFFFu >> (uint32_t)(b + 32 - e_hi);
  return m;
}

// 'N' suppression of the AVX2 path (src/avx2_seeding.rs:115-126,179): window e of quarter-lane l = (e-20)/q is
// suppressed iff some base p in [max(e-20, l*q+20), e] is 'N' (the 20-base prefill of each lane never looks for N).
// nm_lo / nm_hi = N-masks of units u-1 / u (bit b = base b of the unit).  Returns the mask of suppressed windows.
SK_HD uint32_t unit_n_suppress_mask(uint32_t n, uint32_t ul, uint32_t nm_lo, uint32_t nm_hi, uint32_t cand) {
  uint64_t nm = ((uint64_t)nm_hi << 32) | nm_lo;  // relative base r = p - 32*(ul-1), bit r
  if (nm == 0 || cand == 0) return 0;
  uint32_t q = (n - 20) / 4;
  uint32_t sup = 0;
  for (uint32_t j = 0; j < 32; j++) {
    if (!((cand >> j) & 1u)) continue;
    int64_t e = 32ll * ul + j;
    int64_t lane = (e - 20) / (int64_t)q;  // cand only holds existing windows, so q > 0 and 0 <= lane <= 3
    int64_t lb = e - 20;
    int64_t lane_lb = lane * (int64_t)q + 20;
    if (lane_lb > lb) lb = lane_lb;
    // relative indices
    int64_t base0 = 32ll * ((int64_t)ul - 1);
    uint32_t r_lo = (uint32_t)(lb - base0), r_hi = (uint32_t)(e - base0);  // 12 <= r_lo <= r_hi <= 63
    uint64_t span = (r_hi - r_lo == 63) ? ~0ull : (((1ull << (r_hi - r_lo + 1)) - 1) << r_lo);
    if (nm & span) sup |= 1u << j;
  }
  return sup;
}

// ---- scalar seeding semantics (fmh_seeds, src/seeding.rs:225-323: what the reference runs on hosts WITHOUT AVX2) ----
// one lane over the whole contig: every window end e with 20 <= e < n exists (no quarter-lane tail drop); n < 42 -> none
SK_HD uint32_t unit_valid_mask_scalar(uint32_t n, uint32_t ul) {
  if (n < 2 * MARKER_K) return 0;
  const uint64_t e_lo = 20, e_hi = n;
  const uint64_t b = 32ull * ul;
  uint32_t m = 0xFFFFFFFFu;
  if (b + 32 <= e_lo || b >= e_hi) return 0;
  if (b < e_lo) m &= 0xFFFFFFFFu << (uint32_t)(e_lo - b);
  if (b + 32 > e_hi) m &= 0xFFFFFFFFu >> (uint32_t)(b + 32 - e_hi);
  return m;
}
// 'N' / 'n' at position p >= 20 sets resume_ind = p + k (src/seeding.rs:273-275): window e is suppressed iff such a byte lies in
// [max(e - k + 1, 20), e].  The mask bits must flag 'N' AND 'n' (pack_word(..., small_n = true)).
SK_HD uint32_t unit_n_suppress_mask_scalar(uint32_t ul, uint32_t k, uint32_t nm_lo, uint32_t nm_hi, uint32_t cand) {
  const uint64_t nm = ((uint64_t)nm_hi << 32) | nm_lo;   // relative base r = p - 32*(ul-1), bit r
  if (nm == 0 || cand == 0) return 0;
  uint32_t sup = 0;
  for (uint32_t j = 0; j < 32; j++) {
    if (!((cand >> j) & 1u)) continue;
    const int64_t e = 32ll * ul + j;
    int64_t lb = e - (int64_t)k + 1;
    if (lb < 20) lb = 20;
    const int64_t base0 = 32ll * ((int64_t)ul - 1);
    const uint32_t r_lo = (uint32_t)(lb - base0), r_hi = (uint32_t)(e - base0);   // e >= 20 and k <= 16: 17 <= r_lo <= r_hi <= 63
    const uint64_t span = (((r_hi - r_lo == 63) ? ~0ull : ((1ull << (r_hi - r_lo + 1)) - 1)) << r_lo);
    if (nm & span) sup |= 1u << j;
  }
  return sup;
}

}  // namespace sk

namespace sk {

// FracMinHash pass mask of one unit: bit j set iff window j exists, hash(seed) < threshold (src/avx2_seeding.rs:179
// `v < threshold_unsigned`) and the window is not 'N'-suppressed.
SK_HD uint32_t unit_pass_mask(uint64_t lo, uint64_t hi, uint32_t nm_lo, uint32_t nm_hi, uint32_t n, uint32_t ul,
                              uint64_t seed_mask, uint64_t threshold) {
  uint32_t valid = unit_valid_mask(n, ul);
  if (valid == 0) return 0;
  WindowCtx w = make_window_ctx(lo, hi);
  uint32_t pass = 0;
#if defined(__CUDA_ARCH__)
#pragma unroll
#endif
  for (uint32_t j = 0; j < 32; j++) {
    uint64_t fs = window_f21(w, j) & seed_mask;
    uint64_t rs = window_r21(w, j) & seed_mask;
    uint64_t seed = fs < rs ? fs : rs;
    if (mm_hash64(seed) < threshold) pass |= 1u << j;
  }
  pass &= valid;
  if ((nm_lo | nm_hi) != 0 && pass != 0) pass &= ~unit_n_suppress_mask(n, ul, nm_lo, nm_hi, pass);
  return pass;
}

}  // namespace sk

namespace sk {

// ---- tuned variant of unit_pass_mask used by hashpass_kernel: 32-bit seed extraction, multiply-form hash ----------
SK_HD uint32_t funnel_r32(uint32_t lo, uint32_t hi, uint32_t sh) {  // low 32 bits of (hi:lo) >> sh, 0 <= sh <= 31
#if defined(__CUDA_ARCH__)
  return __funnelshift_r(lo, hi, sh);
#else
  return sh ? (lo >> sh) | (hi << (32 - sh)) : lo;
#endif
}
// mm_hash64 with its shift-add steps written as multiplications (x + (x << s) == x * (2^s + 1) mod 2^64): the
// 64-bit multiplies issue on the FMA pipe (IMAD) and relieve the ALU pipe (LOP3/SHF/IADD3) that bounds the kernel.
SK_HD uint64_t mm_hash64_mul(uint64_t key) {
  // steps 1 + 2, x = ~(key * 0x200001); x ^= x >> 24, with the complement folded into the xors (two LOP3 fewer per window):
  //   low word : ~a ^ ~f == a ^ f                         (f = the funnel-shifted low word of the un-complemented product)
  //   high word: ~b ^ ((~b) >> 24) == b ^ (b >> 24) ^ 0xFFFFFF00
  {
    const uint64_t k = key * 0x200001ull;
    const uint32_t a = (uint32_t)k, b = (uint32_t)(k >> 32);
    const uint32_t lo = a ^ funnel_r32(a, b, 24);
    const uint32_t hi = b ^ (b >> 24) ^ 0xFFFFFF00u;
    key = ((uint64_t)hi << 32) | lo;
  }
  key = key * 265ull;
  key = key ^ (key >> 14);
  key = key * 21ull;
  key = key ^ (key >> 28);
  key = key * 0x80000001ull;
  return key;
}

SK_HD uint32_t unit_pass_mask_fast(uint64_t lo, uint64_t hi, uint32_t nm_lo, uint32_t nm_hi, uint32_t n, uint32_t ul,
                                   uint32_t seed_mask32, uint64_t threshold, uint32_t scalar_k = 0) {
  // scalar_k != 0: scalar fmh_seeds semantics (src/seeding.rs:225-323) with that k; 0 = avx2_fmh_seeds (the default)
  const uint32_t valid = scalar_k ? unit_valid_mask_scalar(n, ul) : unit_valid_mask(n, ul);
  if (valid == 0) return 0;
  const uint64_t clo = ~lo, chi = ~hi;
  const uint64_t tlo = pair_reverse64(hi), thi = pair_reverse64(lo);
  const uint32_t c[4] = {(uint32_t)clo, (uint32_t)(clo >> 32), (uint32_t)chi, (uint32_t)(chi >> 32)};
  const uint32_t t[4] = {(uint32_t)tlo, (uint32_t)(tlo >> 32), (uint32_t)thi, (uint32_t)(thi >> 32)};
  uint32_t pass = 0;
#if defined(__CUDA_ARCH__)
#pragma unroll
#endif
  for (uint32_t j = 0; j < 32; j++) {
    const uint32_t orv = 24 + 2 * j;   // bit offset of the reverse seed in the complemented stream (<= 86; + 32 bits <= 118)
    const uint32_t ofw = 62 - 2 * j;   // bit offset of the forward seed in the pair-reversed stream (<= 62)
    const uint32_t rs = funnel_r32(c[orv >> 5], c[(orv >> 5) + 1], orv & 31) & seed_mask32;
    const uint32_t fs = funnel_r32(t[ofw >> 5], t[(ofw >> 5) + 1], ofw & 31) & seed_mask32;
    const uint32_t seed = fs < rs ? fs : rs;
    if (mm_hash64_mul((uint64_t)seed) < threshold) pass |= 1u << j;
  }
  pass &= valid;
  if ((nm_lo | nm_hi) != 0 && pass != 0)
    pass &= ~(scalar_k ? unit_n_suppress_mask_scalar(ul, scalar_k, nm_lo, nm_hi, pass) : unit_n_suppress_mask(n, ul, nm_lo, nm_hi, pass));
  return pass;
}

}  // namespace sk

namespace sk {

// ---- marker screen predicate (screen_rows_kernel, ts_rows_kernel) -----------------------------------------------------
// Modes 0-3 are the query x ref screens of sk_screen_query_ref; the triangle screens with screen_refs' rule.
enum ScreenMode { MODE_QUICK = 0, MODE_QUICK_NORESCUE = 1, MODE_INDEX = 2, MODE_INDEX_NORESCUE = 3, MODE_TRIANGLE = 4 };
constexpr uint64_t SCREEN_MINIMUM_KMERS = 20;   // reference src/params.rs:49

// screen_refs (triangle, mode 2): a row (the screen_refs query) with < 20 markers passes every column when rescue is on
// (src/screen.rs:158-160).  Only the row's own count decides; a small column never rescues its row.
SK_HD bool screen_row_rescued(int mode, bool rescue_small, uint64_t card_row) {
  return (mode == MODE_TRIANGLE || mode == MODE_INDEX) && rescue_small && card_row < SCREEN_MINIMUM_KMERS;
}

// Whether the pair (row, column) passes, given the markers they share (`count`) and cutoff = screen_val^21 (screen_val 0
// already replaced by 0.80, as every caller of the reference does).
SK_HD bool screen_pass(int mode, bool rescue_small, uint64_t card_row, uint64_t card_col, uint64_t count, double cutoff) {
  const uint64_t mn = card_row < card_col ? card_row : card_col;
  if (mode == MODE_TRIANGLE || mode == MODE_INDEX || mode == MODE_INDEX_NORESCUE) {
    // screen_refs / screen_refs_indices (src/screen.rs:177-187, 63-73): only columns with >= 1 shared marker are candidates;
    // pass iff count > max((usize)(cutoff * min(|Mj|,|Mi|)), 1)
    if (screen_row_rescued(mode, rescue_small, card_row)) return true;
    unsigned long long thr = (unsigned long long)(cutoff * (double)mn);
    if (thr < 1) thr = 1;
    return count > thr;
  }
  // check_markers_quickly (src/screen.rs:84-142): symmetric in its two sketches, rescue only in mode 0
  const bool rescue = (mode == MODE_QUICK) && rescue_small;
  if (mn < SCREEN_MINIMUM_KMERS && rescue) return true;
  if (mn == 0) return rescue;
  unsigned long long ratio = (unsigned long long)(cutoff * (double)mn);
  if (ratio == 0) ratio = 1;
  return count >= ratio;
}

}  // namespace sk

