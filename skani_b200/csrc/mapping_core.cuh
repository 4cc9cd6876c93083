// mapping_core.cuh -- per-record logic of sk_chain_pairs_mappings (chain.cu: mapping_emit_kernel) as __host__ __device__
// functions, so that the same code runs inside the kernel and inside tests/emu/emu_mappings.cpp on the host (see sk_core.cuh).
//
// A mapping record is one chain interval that the non-overlap selection kept, in the caller's orientation, joined to the
// identity estimate of the chunk it was chained in.
#pragma once
#include <stdint.h>

#include "../../include/skani_b200.h"
#include "chain_core.cuh"

namespace sk {

static_assert(sizeof(sk_mapping) == 48, "sk_mapping is mirrored by ctypes, numpy and Rust: 48 bytes");

// The record of kept interval x of a pair.  switched: switch_qr chained the caller's reference in the query role, so the
// interval's query side is the caller's reference and its chunks are windows of the reference; the sides are swapped back.
// valid: chunkstat_kernel's chunk_valid (0 no estimate, 1 estimate, 3 estimate after the putative-ANI filter); est / weight
// are only read when valid != 0, and are 0 otherwise.
SK_HD sk_mapping mapping_record(const IntervalKey& x, bool switched, double est, uint32_t weight, uint8_t valid) {
  sk_mapping m;
  const uint32_t q0 = iv_q0(x), q1 = iv_q1(x), r0 = iv_r0(x), r1 = iv_r1(x), qc = iv_qctg(x), rc = iv_rctg(x);
  m.query_contig = switched ? rc : qc; m.ref_contig = switched ? qc : rc;
  m.q0 = switched ? r0 : q0; m.q1 = switched ? r1 : q1;
  m.r0 = switched ? q0 : r0; m.r1 = switched ? q1 : r1;
  m.num_anchors = iv_num_anchors(x); m.chunk = iv_chunk(x);
  m.chunk_est = valid ? est : 0.;
  m.chunk_weight = valid ? weight : 0u;
  m.reverse = (uint8_t)iv_rev(x); m.switched = switched ? 1 : 0; m.chunk_valid = valid; m.pad = 0;
  return m;
}

// The order of a pair's records: (query_contig, q0, q1, ref_contig, r0, r1, reverse, chunk), ascending.
SK_HD bool mapping_before(const sk_mapping& a, const sk_mapping& b) {
  if (a.query_contig != b.query_contig) return a.query_contig < b.query_contig;
  if (a.q0 != b.q0) return a.q0 < b.q0;
  if (a.q1 != b.q1) return a.q1 < b.q1;
  if (a.ref_contig != b.ref_contig) return a.ref_contig < b.ref_contig;
  if (a.r0 != b.r0) return a.r0 < b.r0;
  if (a.r1 != b.r1) return a.r1 < b.r1;
  if (a.reverse != b.reverse) return a.reverse < b.reverse;
  return a.chunk < b.chunk;
}

}  // namespace sk
