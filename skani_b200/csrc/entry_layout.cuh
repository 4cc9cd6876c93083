// entry_layout.cuh -- where each section of a skani v0.3 sketch entry lies, as skdb::put_params + skdb::put_sketch
// (cli/sketch_db.hpp) write it, from the counts alone.  __host__ __device__: sk_sketch_set_encode lays entries out on the
// host and its kernels write the records, lists and markers at these offsets.
//   full entry      (SketchParams, Sketch)          one sketches.db entry, or a whole .sketch file
//   markers-only    Sketch::get_markers_only        one element of markers.bin's Vec<Sketch> (no params, no seeds,
//                                                   no contig lengths)
#pragma once
#include <stdint.h>

#include "sketch_value.cuh"

namespace skdb {

constexpr uint64_t PARAMS_BYTES = 3 * 8 + 2 + 8 + 64 * 8 + 8 + 64 + 8;   // put_params: 626
constexpr uint64_t TAIL_BYTES = 4 * 8 + 2;                              // marker_c, c, k, contig_order, two flags

// What one entry holds.  n_multi: keys with two or more records; the multi-position lists then take
// 8 + 8 * n_multi + 8 * (n_records - n_keys + n_multi) bytes, their length prefixes included.
struct EntryCounts {
  bool params = true, seeds = true;    // full entry: both; markers-only: neither
  uint64_t name_len = 0;               // bytes of file_name
  uint64_t n_keys = 0, n_records = 0, n_multi = 0;
  uint64_t n_contigs = 0, contig_name_bytes = 0;   // contig names and the sum of their lengths
  uint64_t n_contig_lengths = 0;
  uint64_t n_markers = 0;
};

// byte offsets from the entry's first byte; each *_at names the section's first byte (a length prefix where it has one)
struct EntryLayout {
  uint64_t name_at;        // u64 length + file_name
  uint64_t tag_at;         // Option tag of kmer_seeds_k
  uint64_t keys_at;        // full: u64 n_keys, then n_keys x {u32 k-mer, u64 value}
  uint64_t multi_at;       // u64 n_multi, then per list u64 length + length x {u32 pos, u32 contig_index_canonical}
  uint64_t contigs_at;     // u64 count, then per name u64 length + bytes
  uint64_t total_len_at;   // u64
  uint64_t ctg_len_at;     // u64 count, then u32 each
  uint64_t repetitive_at;  // u64
  uint64_t markers_at;     // u64 count, then u64 each
  uint64_t tail_at;        // TAIL_BYTES
  uint64_t length;
};

SK_HD EntryLayout entry_layout(const EntryCounts& c) {
  EntryLayout l;
  l.name_at = c.params ? PARAMS_BYTES : 0;
  l.tag_at = l.name_at + 8 + c.name_len;
  l.keys_at = l.tag_at + 1;
  l.multi_at = c.seeds ? l.keys_at + 8 + 12 * c.n_keys : l.keys_at;
  l.contigs_at = l.multi_at + 8 + (c.seeds ? 8 * c.n_multi + 8 * (c.n_records - c.n_keys + c.n_multi) : 0);
  l.total_len_at = l.contigs_at + 8 + 8 * c.n_contigs + c.contig_name_bytes;
  l.ctg_len_at = l.total_len_at + 8;
  l.repetitive_at = l.ctg_len_at + 8 + 4 * c.n_contig_lengths;
  l.markers_at = l.repetitive_at + 8;
  l.tail_at = l.markers_at + 8 + 8 * c.n_markers;
  l.length = l.tail_at + TAIL_BYTES;
  return l;
}

}  // namespace skdb
