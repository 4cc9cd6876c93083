// derep_core.cuh -- per-pair logic of sk_dereplicate (derep.cu) as __host__ __device__ functions, so that the same code
// runs inside the CUDA kernels and inside tests/emu/emu_derep.cpp on the host (see sk_core.cuh).
//
// The representative index holds keys marker << DR_SLOT_BITS | slot: the slot is the dense number of a representative (or,
// for the screen inside a wave, of an undecided wave genome), so a run of equal markers lists the slots that hold it.
#pragma once
#include <stdint.h>

#include "sk_core.cuh"

namespace sk {

constexpr uint32_t DR_SLOT_BITS = 22;                       // slot bits of an index key: at most 2^22 - 1 slots
constexpr uint32_t DR_MAX_SLOTS = (1u << DR_SLOT_BITS) - 1;
constexpr uint64_t DR_MAX_KEYS = 1ull << 31;                // index entries (one per marker of a slot) must stay below this
constexpr uint32_t DR_PREFIX_BITS = 16;
constexpr uint32_t DR_PREFIX_SHIFT = 2 * MARKER_K + DR_SLOT_BITS - DR_PREFIX_BITS;

SK_HD uint64_t dr_key(uint64_t marker, uint32_t slot) { return marker << DR_SLOT_BITS | slot; }
SK_HD uint32_t dr_key_slot(uint64_t key) { return (uint32_t)(key & DR_MAX_SLOTS); }
SK_HD uint64_t dr_key_marker(uint64_t key) { return key >> DR_SLOT_BITS; }

// the key of the unordered pair {a, b} as the triangle chains it: min << 32 | max
SK_HD uint64_t dr_pair_key(uint32_t a, uint32_t b) { return a < b ? (uint64_t)a << 32 | b : (uint64_t)b << 32 | a; }

// The triangle's screen decision for genomes a != b with card_a / card_b markers and `count` shared ones.  sk_screen_triangle
// decides the pair (i, j), i < j, with row i (screen_refs with the smaller genome INDEX as its query, src/screen.rs:158-160):
// only the smaller index's marker count can rescue the pair, whatever the two genomes' ranks or which one is the
// representative.
SK_HD bool dr_screen_pass(uint32_t a, uint64_t card_a, uint32_t b, uint64_t card_b, uint64_t count, bool rescue_small, double cutoff) {
  return a < b ? screen_pass(MODE_TRIANGLE, rescue_small, card_a, card_b, count, cutoff)
               : screen_pass(MODE_TRIANGLE, rescue_small, card_b, card_a, count, cutoff);
}

}  // namespace sk
