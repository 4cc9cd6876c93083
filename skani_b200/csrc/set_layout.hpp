// set_layout.hpp -- the device arrays of a sketch set, described once.  Host-only (no CUDA header).
//
// A sketch set (sk_sketch_set, sk_internal.h) is the twelve arrays of SET_ARRAYS.  Each is counted by one of the set's
// prefix offsets: records S (seed_off), distinct k-mers U (uk_off), markers M (mk_off), contigs C (ctg_off) or k-mer table
// slots HT (ht_off).  Two of them carry one sentinel per genome, so genome i's slice starts at prefix[i] + i.  A blob
// (sk_sketch_set_pack_subset / sk_sketch_set_unpack, the host sketch store) holds the arrays in table order, each 256-byte
// aligned; its host metadata is the word vector of encode_meta.  Everything that moves a set walks this table.
#pragma once
#include <stddef.h>
#include <stdint.h>

#include <vector>

namespace sk {

enum Count : int { CNT_S, CNT_U, CNT_M, CNT_C, CNT_HT, N_COUNTS };   // also the order of the offset vectors in the metadata

struct ArrayDesc {
  const char* name;
  uint32_t esz;       // element bytes
  Count by;           // the prefix the array is counted by
  bool sentinel;      // one extra element per genome
  bool markers_only;  // travels in SK_PACK_MARKERS_ONLY blobs (there the others are empty, and the sentinels are zero)
  bool tables_only;   // travels only with SK_PACK_TABLES
};

constexpr int BLOB_ARRAYS = 12;
constexpr ArrayDesc SET_ARRAYS[BLOB_ARRAYS] = {
    {"pv_kmer", 4, CNT_S, false, false, false},     {"pv_pos", 4, CNT_S, false, false, false},  {"pv_cc", 4, CNT_S, false, false, false},
    {"pv_mult", 2, CNT_S, false, false, false},     {"kv_pos", 4, CNT_S, false, false, false},  {"kv_cc", 4, CNT_S, false, false, false},
    {"ukmer", 4, CNT_U, false, false, false},       {"ustart", 4, CNT_U, true, false, false},   {"markers", 8, CNT_M, false, true, false},
    {"ctg_rec_off", 4, CNT_C, true, false, false},  {"d_ctg_len", 4, CNT_C, false, false, false}, {"htab", 8, CNT_HT, false, false, true}};
constexpr int HTAB_ARRAY = 11;
static_assert(SET_ARRAYS[HTAB_ARRAY].by == CNT_HT, "htab is the table-slot array");

// elements of array a for G genomes with totals n
inline uint64_t array_elems(int a, uint64_t G, const uint64_t n[N_COUNTS]) { return n[SET_ARRAYS[a].by] + (SET_ARRAYS[a].sentinel ? G : 0); }
// element index of genome i's slice in a concatenation, given prefix[i] of the array's count
inline uint64_t array_index(int a, uint64_t i, uint64_t prefix_i) { return prefix_i + (SET_ARRAYS[a].sentinel ? i : 0); }
inline bool array_travels(int a, bool markers_only, bool tables) {
  return markers_only ? SET_ARRAYS[a].markers_only : (tables || !SET_ARRAYS[a].tables_only);
}
// a count is non-zero in a blob only when an array counted by it travels
inline bool count_travels(Count x, bool markers_only, bool tables) {
  for (int a = 0; a < BLOB_ARRAYS; a++)
    if (SET_ARRAYS[a].by == x && array_travels(a, markers_only, tables)) return true;
  return false;
}

inline size_t al256(size_t x) { return (x + 255) & ~(size_t)255; }

struct BlobLayout {
  size_t off[BLOB_ARRAYS];
  size_t bytes[BLOB_ARRAYS];
  size_t total;
};
inline BlobLayout blob_layout(uint64_t G, const uint64_t n[N_COUNTS]) {
  BlobLayout b;
  size_t o = 0;
  for (int a = 0; a < BLOB_ARRAYS; a++) { b.off[a] = o; b.bytes[a] = array_elems(a, G, n) * SET_ARRAYS[a].esz; o += al256(b.bytes[a]); }
  b.total = o ? o : 256;
  return b;
}

// a genome's record in the host sketch store: its arrays back to back, each slice 16-byte aligned; returns the record bytes
inline uint64_t genome_slices(const uint64_t n[N_COUNTS], uint64_t slice[BLOB_ARRAYS]) {
  uint64_t o = 0;
  for (int a = 0; a < BLOB_ARRAYS; a++) { slice[a] = o; o += (array_elems(a, 1, n) * SET_ARRAYS[a].esz + 15) & ~15ull; }
  return o;
}
// device bytes of one genome in a set (= 22 S + 8 U + 8 M + 8 C + 8 HT + 8)
inline uint64_t genome_bytes(const uint64_t n[N_COUNTS]) {
  uint64_t b = 0;
  for (int a = 0; a < BLOB_ARRAYS; a++) b += array_elems(a, 1, n) * SET_ARRAYS[a].esz;
  return b;
}

// host metadata of a blob.  Words: META_HEADER = G S U M C c k marker_c HT tables, then seed_off uk_off mk_off ctg_off
// [G+1 each], total_len [G], the contig lengths [C] genome-major and, with tables, ht_off [G+1]
constexpr int META_HEADER = 10;
struct SetMeta {
  uint64_t G = 0;
  uint64_t n[N_COUNTS] = {};             // totals S U M C HT
  uint64_t c = 0, k = 0, marker_c = 0;   // sketch parameters
  bool tables = false;
  std::vector<uint64_t> off[N_COUNTS] = {{0}, {0}, {0}, {0}, {0}};   // prefix offsets [G+1]; ht_off all zero without tables
  std::vector<uint64_t> total_len;       // [G]
  std::vector<uint64_t> ctg_len;         // [C]
};
inline uint64_t meta_words(uint64_t G, uint64_t C, bool tables) { return META_HEADER + 4 * (G + 1) + G + C + (tables ? G + 1 : 0); }

// appends a genome with counts n to a blob's metadata (set c, k, marker_c and tables first): the counts of arrays that do not
// travel become 0, and a markers-only blob keeps no contig lengths
template <class It>
inline void meta_push(SetMeta& m, const uint64_t n[N_COUNTS], bool markers_only, uint64_t total_len, It ctg_begin, It ctg_end) {
  for (int x = 0; x < N_COUNTS; x++) {
    const uint64_t v = count_travels((Count)x, markers_only, m.tables) ? n[x] : 0;
    m.off[x].push_back(m.off[x].back() + v);
    m.n[x] += v;
  }
  m.G++;
  m.total_len.push_back(total_len);
  if (!markers_only) m.ctg_len.insert(m.ctg_len.end(), ctg_begin, ctg_end);
}

inline void encode_meta(const SetMeta& m, uint64_t* w) {
  for (uint64_t x : {m.G, m.n[CNT_S], m.n[CNT_U], m.n[CNT_M], m.n[CNT_C], m.c, m.k, m.marker_c, m.n[CNT_HT], (uint64_t)m.tables}) *w++ = x;
  for (int x = CNT_S; x <= CNT_C; x++) for (uint64_t v : m.off[x]) *w++ = v;
  for (uint64_t v : m.total_len) *w++ = v;
  for (uint64_t v : m.ctg_len) *w++ = v;
  if (m.tables) for (uint64_t v : m.off[CNT_HT]) *w++ = v;
}
inline SetMeta decode_meta(const uint64_t* w) {
  SetMeta m;
  m.G = w[0];
  m.n[CNT_S] = w[1]; m.n[CNT_U] = w[2]; m.n[CNT_M] = w[3]; m.n[CNT_C] = w[4];
  m.c = w[5]; m.k = w[6]; m.marker_c = w[7]; m.n[CNT_HT] = w[8]; m.tables = w[9] != 0;
  w += META_HEADER;
  for (int x = CNT_S; x <= CNT_C; x++) { m.off[x].assign(w, w + m.G + 1); w += m.G + 1; }
  m.total_len.assign(w, w + m.G); w += m.G;
  m.ctg_len.assign(w, w + m.n[CNT_C]); w += m.n[CNT_C];
  if (m.tables) m.off[CNT_HT].assign(w, w + m.G + 1);
  else m.off[CNT_HT].assign(m.G + 1, 0);
  return m;
}

}  // namespace sk
