// sketch_value.cuh -- the value of a skani v0.3 k-mer map entry (src/types.rs:207-244), as __host__ __device__ inline
// functions: the host decoder (cli/sketch_db.hpp) and the device expansion of sk_sketch_set_import_blobs read it alike.
//   bit 0 = 1: one position, ((pos << 31 | contig_index_canonical) << 1) | 1
//   bit 0 = 0: (index into multi_position_storage) << 1
#pragma once
#include <stdint.h>

#ifndef SK_HD
#if defined(__CUDACC__)
#define SK_HD __host__ __device__ __forceinline__
#else
#define SK_HD inline
#endif
#endif

namespace skdb {

SK_HD bool value_is_single(uint64_t v) { return (v & 1) != 0; }
SK_HD uint32_t value_pos(uint64_t v) { return (uint32_t)(v >> 32); }                    // ((v >> 1) >> 31)
SK_HD uint32_t value_cc(uint64_t v) { return (uint32_t)((v >> 1) & 0x7FFFFFFFull); }
SK_HD uint64_t value_multi_index(uint64_t v) { return v >> 1; }
SK_HD uint64_t single_value(uint32_t pos, uint32_t cc) { return ((((uint64_t)pos << 31) | (uint64_t)cc) << 1) | 1ull; }
SK_HD uint64_t multi_value(uint64_t index) { return index << 1; }

}  // namespace skdb
