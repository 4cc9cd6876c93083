// Host emulation of sk_chain_pairs_mappings' per-record logic (skani_b200/csrc/mapping_core.cuh: mapping_record, the
// un-switching and chunk join, and mapping_before, the order of a pair's records, as mapping_emit_kernel applies them) on
// the CPU oracle's chain taps.  Development/test harness only; not a product path.
//
// usage: emu_mappings c robust median learned_ani file_a file_b
// Sketches both files with the oracle, runs chain_seeds on (ref a, query b) and (ref b, query a) with the debug taps, turns
// every kept interval into a record with its chunk's chunk_estimate and sorts the pair's records.  Prints, per pair, a line
// "PAIR <ref> <query> <n>" and then one line per record: query_contig ref_contig q0 q1 r0 r1 num_anchors chunk
// chunk_est (%a) chunk_weight reverse switched chunk_valid.
#include <cstdio>
#include <cstdlib>
#include <algorithm>
#include <string>
#include <vector>

#include "../../skani_b200/csrc/mapping_core.cuh"
#include "../../oracle/skani_oracle.hpp"

int main(int argc, char** argv) {
  if (argc != 7) { fprintf(stderr, "usage: emu_mappings c robust median learned_ani file_a file_b\n"); return 2; }
  orc::SketchParams sp{};
  sp.c = (uint32_t)atoi(argv[1]); sp.k = 15; sp.marker_c = 1000;
  orc::CommandParams cp;
  cp.robust = atoi(argv[2]) != 0; cp.median = atoi(argv[3]) != 0; cp.learned_ani = atoi(argv[4]) != 0;
  std::vector<orc::Sketch> sk = orc::fastx_to_sketches({argv[5], argv[6]}, sp, false, true, 2, nullptr);
  if (sk.size() != 2) { fprintf(stderr, "expected two genomes, got %zu\n", sk.size()); return 1; }
  for (int o = 0; o < 2; o++) {
    const orc::Sketch& ref = sk[o];
    const orc::Sketch& qry = sk[1 - o];
    const orc::MapParams mp = orc::map_params_from_sketch(ref, cp, orc::get_model_id(ref.c, cp.learned_ani));
    orc::ChainDebug dbg;
    orc::chain_seeds(ref, qry, mp, &dbg);
    std::vector<sk_mapping> recs;
    for (size_t i = 0; i < dbg.intervals_all.size(); i++) {
      if (!dbg.interval_kept[i]) continue;
      const orc::ChainInterval& c = dbg.intervals_all[i];
      const uint32_t* st = dbg.chunk_stats.data() + 9 * c.chunk_id;
      orc::ChunkStats s;
      s.total_anchors = st[0]; s.rq0 = st[1]; s.rq1 = st[2]; s.tbcq = st[3]; s.n_int = st[4];
      s.n_seeds = st[5]; s.num_in = st[6]; s.upper_lower = st[7];
      orc::chunk_estimate(s, sp.c, sp.k, orc::MIN_LENGTH_COVER);
      const uint8_t valid = s.valid ? (s.filtered ? 3 : 1) : 0;
      const sk::IntervalKey x = sk::make_interval((int32_t)c.score, (uint32_t)c.num_anchors, c.q0, c.q1, c.r0, c.r1,
                                                  (uint32_t)c.ref_contig, (uint32_t)c.query_contig, (uint32_t)c.chunk_id,
                                                  c.reverse_chain ? 1u : 0u);
      recs.push_back(sk::mapping_record(x, dbg.switched, s.est, (uint32_t)s.weight, valid));
    }
    std::sort(recs.begin(), recs.end(), sk::mapping_before);
    printf("PAIR %d %d %zu\n", o, 1 - o, recs.size());
    for (const sk_mapping& m : recs)
      printf("%u %u %u %u %u %u %u %u %a %u %u %u %u\n", m.query_contig, m.ref_contig, m.q0, m.q1, m.r0, m.r1, m.num_anchors,
             m.chunk, m.chunk_est, m.chunk_weight, m.reverse, m.switched, m.chunk_valid);
  }
  return 0;
}
