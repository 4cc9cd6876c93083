// Host emulation of dp_group_kernel<GL, NE, FULLBAND> (skani_b200/csrc/chain.cu) with its chain bookkeeping where the kernel
// keeps it, checked against the oracle (chain_chunks) on the constructed chunks of tests/dp_select_cases.py and on chunks
// around the on-chip bound.  Development/test harness only, not a product path.  tests/emu/emu_dp_select.cpp emulates the
// candidate evaluation and selection as well; this file mirrors the kernel's bookkeeping and emission:
//
// The 32 / GL groups of a warp run in lockstep, block by block, as the warp's lanes do.  A chunk of at most DP_SMEM_ANCHORS
// anchors keeps one packed word per anchor, score << 16 | index << 8 | (depth - 1), in its group's slab of the warp's shared
// memory (group w's words at w * DP_SMEM_ANCHORS): the word starts as (0, index, 0), a chained anchor atomicMax-es its word
// into its root's, and the emission decodes chain end, score and depth from the root's word once every group's loop is done.
// Longer chunks keep the global rootkey (score << 32 | index, atomicMax) and depth arrays.  A chunk one anchor too long for
// its slab writes into its neighbour's, as it would in the kernel.
//
// Input (stdin, whitespace separated):  D GL NE FULLBAND band c n_chunks { n { qctg qpos rctg rpos rev } }
#include <algorithm>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <string>
#include <vector>

#include "../../skani_b200/csrc/chain_core.cuh"
#include "../../oracle/skani_oracle.hpp"

using namespace sk;

// dp_group_kernel's on-chip bound (chain.cu); tests/test_emu_dp_onchip.py compares it with the kernel source
constexpr uint32_t DP_SMEM_ANCHORS = 224;

static int failures = 0;
static std::string g_tag;
#define FAIL(...) do { failures++; if (failures <= 20) { fprintf(stdout, "FAIL %s: ", g_tag.c_str()); fprintf(stdout, __VA_ARGS__); fprintf(stdout, "\n"); } } while (0)

static long n_dp_configs, n_chunks_onchip, n_chunks_global, n_anchors_all, n_iv_all;

struct Chunk { uint32_t qctg; std::vector<AnchorRec> a; };

static bool in_band(uint32_t d, uint32_t band) { return d <= band; }
static bool dq_ok(uint32_t dq) { return dq - 1u < BP_CHAIN_BAND; }
static bool dr_ok(uint32_t dr) { return dr - 1u < (uint32_t)MAX_LIN; }
static bool gap_ok(uint32_t g) { return g + (uint32_t)MAX_GAP <= 2u * (uint32_t)MAX_GAP; }

// onchip: the chunk's bookkeeping is the packed word per anchor, else the global rootkey / depth arrays (key, depth)
struct DpOut { std::vector<int32_t> score; std::vector<uint32_t> ptr, depth, word; std::vector<unsigned long long> key; bool onchip = false; };

static void atomic_max(unsigned long long& x, unsigned long long v) { if (v > x) x = v; }
static void atomic_max32(uint32_t& x, uint32_t v) { if (v > x) x = v; }

// one warp = 32 / GL chunks (indices into `cs`), nmax = the longest of them
static void dp_group_warp(const std::vector<const Chunk*>& cs, int GL, int NE, bool FULLBAND, uint32_t band, std::vector<DpOut*>& outs) {
  const int NB = NE + 1, LG = GL == 8 ? 3 : 2;
  const size_t GW = 32 / GL;
  uint32_t nmax = 0;
  for (auto* c : cs) nmax = std::max<uint32_t>(nmax, (uint32_t)c->a.size());
  std::vector<uint32_t> s_chain(GW * DP_SMEM_ANCHORS, 0xDEADBEEFu);
  auto slab = [&](size_t w, uint32_t i) -> uint32_t* {
    const size_t at = w * DP_SMEM_ANCHORS + i;
    if (at >= s_chain.size()) { FAIL("group %zu anchor %u, field slab: word %zu is past the warp's %zu", w, i, at, s_chain.size()); return nullptr; }
    return &s_chain[at];
  };
  // registers per group, lane and set
  struct Regs { std::vector<std::vector<uint32_t>> q, r, rc, rt, dp; std::vector<std::vector<int32_t>> sc; std::vector<uint32_t> my_ptr; };
  std::vector<Regs> R(cs.size());
  for (size_t w = 0; w < cs.size(); w++) {
    const uint32_t n = (uint32_t)cs[w]->a.size();
    DpOut& O = *outs[w];
    O.score.assign(n, 0); O.ptr.assign(n, 0); O.depth.assign(n, 0); O.key.assign(n, 0); O.word.assign(n, 0);
    O.onchip = n <= DP_SMEM_ANCHORS;
    Regs& g = R[w];
    g.q.assign(GL, std::vector<uint32_t>(NB, 0)); g.r = g.q; g.rc = g.q; g.rt = g.q; g.dp = g.q;
    g.sc.assign(GL, std::vector<int32_t>(NB, 0));
    g.my_ptr.assign(GL, 0);
    for (int l = 0; l < GL; l++) for (int s = 0; s < NB; s++) g.rc[l][s] = 0xFFFFFFFCu;
  }
  for (uint32_t b0 = 0; b0 < nmax; b0 += GL) {
    for (size_t w = 0; w < cs.size(); w++) {
      const Chunk& C = *cs[w];
      DpOut& O = *outs[w];
      const uint32_t n = (uint32_t)C.a.size();
      auto& q = R[w].q; auto& r = R[w].r; auto& rc = R[w].rc; auto& rt = R[w].rt; auto& dp = R[w].dp; auto& sc = R[w].sc; auto& my_ptr = R[w].my_ptr;
      for (int l = 0; l < GL; l++) {
        for (int s = NB - 1; s > 0; s--) { q[l][s] = q[l][s - 1]; r[l][s] = r[l][s - 1]; rc[l][s] = rc[l][s - 1]; rt[l][s] = rt[l][s - 1]; dp[l][s] = dp[l][s - 1]; sc[l][s] = sc[l][s - 1]; }
        const uint32_t idx = b0 + l;
        AnchorRec x; x.qpos = 0; x.rpos = 0; x.rc = 0xFFFFFFFEu;
        if (idx < n) {
          x = C.a[idx];
          if (O.onchip) { if (uint32_t* s = slab(w, idx)) *s = idx << 8; }
          else O.key[idx] = idx;
        }
        q[l][0] = x.qpos; r[l][0] = (x.rc & 1u) ? (0u - x.rpos) : x.rpos; rc[l][0] = x.rc; sc[l][0] = 0; rt[l][0] = idx; dp[l][0] = 1;
        my_ptr[l] = idx;
      }
    }
    for (size_t w = 0; w < cs.size(); w++) {
      auto& q = R[w].q; auto& r = R[w].r; auto& rc = R[w].rc; auto& rt = R[w].rt; auto& dp = R[w].dp; auto& sc = R[w].sc; auto& my_ptr = R[w].my_ptr;
      for (uint32_t m = 0; m < (uint32_t)GL; m++) {
        const uint32_t i = b0 + m;
        const uint32_t cq = q[m][0], cr = r[m][0], crc = rc[m][0];
        int32_t kmax = 0;
        for (int gl = 0; gl < GL; gl++) {
          int32_t best = 0;
          auto eval = [&](uint32_t qs, uint32_t rs, uint32_t rcs, int32_t scs, uint32_t d) {
            const uint32_t dq = cq - qs;
            const uint32_t dr = cr - rs;
            const uint32_t g = dr - dq;
            const bool ok = (FULLBAND || in_band(d, band)) & (rcs == crc) & dq_ok(dq) & dr_ok(dr) & gap_ok(g);
            const int32_t gi = (int32_t)g;
            const int32_t nsm1 = scs + (ANCHOR_SCORE - 1) - (gi < 0 ? -gi : gi);
            const int32_t key = (int32_t)(((uint32_t)nsm1 << 5) | (31u - d));
            best = std::max(best, ok ? key : 0);
          };
          for (int s2 = 1; s2 < NE; s2++) eval(q[gl][s2], r[gl][s2], rc[gl][s2], sc[gl][s2], m + (uint32_t)(GL * s2) - gl);
          const bool lo_set = (uint32_t)gl < m;
          const int se = lo_set ? 0 : NE;
          eval(q[gl][se], r[gl][se], rc[gl][se], sc[gl][se], m - gl + (lo_set ? 0u : (uint32_t)(GL * NE)));
          kmax = std::max(kmax, best);
        }
        const bool has = kmax > 0;
        const int32_t smax = (kmax >> 5) + 1;
        const uint32_t dwin = 31u - ((uint32_t)kmax & 31u);
        const uint32_t jw = i - dwin;
        const int sidx = (int)(b0 >> LG) - (int)(jw >> LG);
        const uint32_t wl = jw & (uint32_t)(GL - 1);
        uint32_t rsel = rt[wl][0], dsel = dp[wl][0];
        for (int s = 1; s < NB; s++) if (sidx == s) { rsel = rt[wl][s]; dsel = dp[wl][s]; }
        if (has) { sc[m][0] = smax; rt[m][0] = rsel; dp[m][0] = dsel + 1; my_ptr[m] = jw; }
      }
    }
    for (size_t w = 0; w < cs.size(); w++) {
      DpOut& O = *outs[w];
      const uint32_t n = (uint32_t)cs[w]->a.size();
      auto& rt = R[w].rt; auto& dp = R[w].dp; auto& sc = R[w].sc; auto& my_ptr = R[w].my_ptr;
      for (int l = 0; l < GL; l++) {
        const uint32_t idx = b0 + l;
        if (idx < n) {
          O.depth[idx] = dp[l][0];
          if (rt[l][0] >= n) { FAIL("anchor %u, field root: %u is outside the chunk of %u", idx, rt[l][0], n); continue; }
          if (rt[l][0] != idx) {
            if (O.onchip) { if (uint32_t* s = slab(w, rt[l][0])) atomic_max32(*s, ((uint32_t)sc[l][0] << 16) | (idx << 8) | (dp[l][0] - 1)); }
            else atomic_max(O.key[rt[l][0]], ((unsigned long long)(uint32_t)sc[l][0] << 32) | idx);
          }
          O.score[idx] = sc[l][0]; O.ptr[idx] = my_ptr[l];
        }
      }
    }
  }
  // the emission reads the slab once every group's loop is done
  for (size_t w = 0; w < cs.size(); w++) {
    DpOut& O = *outs[w];
    if (!O.onchip) continue;
    for (uint32_t i = 0; i < (uint32_t)O.word.size(); i++) { const uint32_t* s = slab(w, i); O.word[i] = s ? *s : 0u; }
  }
}

// the kernel's interval emission (one per surviving root), from the packed words or the global arrays
static void emit_intervals(const Chunk& C, const DpOut& O, uint32_t chunk_id, std::vector<IntervalKey>& iv) {
  const uint32_t n = (uint32_t)C.a.size();
  for (uint32_t i = 0; i < n; i++) {
    uint32_t b, score, num_anchors;
    if (O.onchip) {
      const uint32_t w = O.word[i];
      b = (w >> 8) & 0xFFu; score = w >> 16; num_anchors = (w & 0xFFu) + 1;
      if (b == i) continue;
      if (b >= n) { FAIL("chunk %u anchor %u, field chain end: %u is outside the chunk of %u", chunk_id, i, b, n); continue; }
    } else {
      if (O.depth[i] != 1) continue;
      const unsigned long long key = O.key[i];
      b = (uint32_t)key; score = (uint32_t)(key >> 32);
      if (b == i || b >= n) continue;
      num_anchors = O.depth[b];
    }
    if (num_anchors < MIN_ANCHORS || (int32_t)score < MIN_SCORE) continue;
    const AnchorRec f = C.a[i], l = C.a[b];
    const uint32_t r0 = f.rpos < l.rpos ? f.rpos : l.rpos, r1 = f.rpos < l.rpos ? l.rpos : f.rpos;
    iv.push_back(make_interval((int32_t)score, num_anchors, f.qpos, l.qpos, r0, r1, f.rc >> 1, C.qctg, chunk_id, f.rc & 1u));
  }
}

static const char* IVF[] = {"score", "num_anchors", "q0", "q1", "r0", "r1", "ref_contig", "query_contig", "chunk", "reverse"};
static int64_t ivf(const IntervalKey& x, int f) {
  switch (f) {
    case 0: return (int64_t)iv_score(x); case 1: return (int64_t)iv_num_anchors(x); case 2: return iv_q0(x); case 3: return iv_q1(x);
    case 4: return iv_r0(x); case 5: return iv_r1(x); case 6: return (int64_t)iv_rctg(x); case 7: return (int64_t)iv_qctg(x);
    case 8: return (int64_t)iv_chunk(x); default: return iv_rev(x);
  }
}

static orc::MapParams map_params(uint32_t c, uint32_t k) {
  orc::Sketch unit;
  unit.c = c; unit.k = k;
  return orc::map_params_from_sketch(unit, orc::CommandParams(), -1);
}

static void run_dp(int GL, int NE, bool FULLBAND, uint32_t band, uint32_t c, const std::vector<Chunk>& chunks) {
  n_dp_configs++;
  char tag[128];
  snprintf(tag, sizeof(tag), "dp_group_kernel<GL=%d, NE=%d, FULLBAND=%d> band %u", GL, NE, (int)FULLBAND, band);
  g_tag = tag;
  std::vector<DpOut> outs(chunks.size());
  // the radix sort by descending size is stable: equal sizes keep their chunk order
  std::vector<uint32_t> perm(chunks.size());
  for (uint32_t i = 0; i < perm.size(); i++) perm[i] = i;
  std::stable_sort(perm.begin(), perm.end(), [&](uint32_t a, uint32_t b) { return chunks[a].a.size() > chunks[b].a.size(); });
  const size_t GW = 32 / GL;
  for (size_t w0 = 0; w0 < perm.size(); w0 += GW) {
    std::vector<const Chunk*> cs;
    std::vector<DpOut*> os;
    for (size_t t = w0; t < std::min(perm.size(), w0 + GW); t++) { cs.push_back(&chunks[perm[t]]); os.push_back(&outs[perm[t]]); }
    dp_group_warp(cs, GL, NE, FULLBAND, band, os);
  }
  std::vector<std::vector<orc::Anchor>> oc(chunks.size());
  for (size_t i = 0; i < chunks.size(); i++)
    for (const AnchorRec& a : chunks[i].a) oc[i].push_back(orc::Anchor{chunks[i].qctg, a.qpos, a.rc >> 1, a.rpos, (a.rc & 1u) != 0});
  std::vector<double> osc;
  std::vector<uint32_t> optr;
  std::vector<IntervalKey> oiv;
  for (const orc::ChainInterval& v : orc::chain_chunks(oc, map_params(c, 15), &osc, &optr))
    oiv.push_back(make_interval((int32_t)v.score, (uint32_t)v.num_anchors, (uint32_t)v.q0, (uint32_t)v.q1, (uint32_t)v.r0, (uint32_t)v.r1,
                                (uint32_t)v.ref_contig, (uint32_t)v.query_contig, (uint32_t)v.chunk_id, v.reverse_chain ? 1u : 0u));
  size_t off = 0;
  std::vector<IntervalKey> iv;
  for (size_t i = 0; i < chunks.size(); i++) {
    for (size_t x = 0; x < chunks[i].a.size(); x++) {
      if (outs[i].score[x] != (int32_t)osc[off + x]) { FAIL("chunk %zu anchor %zu, field score: emulated %d, oracle %d", i, x, outs[i].score[x], (int32_t)osc[off + x]); return; }
      if (outs[i].ptr[x] != optr[off + x]) { FAIL("chunk %zu anchor %zu, field pointer: emulated %u, oracle %u", i, x, outs[i].ptr[x], optr[off + x]); return; }
    }
    off += chunks[i].a.size();
    n_anchors_all += chunks[i].a.size();
    (outs[i].onchip ? n_chunks_onchip : n_chunks_global)++;
    emit_intervals(chunks[i], outs[i], (uint32_t)i, iv);
  }
  n_iv_all += iv.size();
  // the emission order is free (select_kernel sorts): compare both lists in the sorted order
  auto before = [](const IntervalKey& a, const IntervalKey& b) { return interval_before(a, b); };
  std::sort(iv.begin(), iv.end(), before);
  std::sort(oiv.begin(), oiv.end(), before);
  if (iv.size() != oiv.size()) { FAIL("%zu intervals emulated, %zu in the oracle", iv.size(), oiv.size()); return; }
  for (size_t i = 0; i < iv.size(); i++)
    for (int f = 0; f < 10; f++)
      if (ivf(iv[i], f) != ivf(oiv[i], f)) { FAIL("interval %zu, field %s: emulated %lld, oracle %lld", i, IVF[f], (long long)ivf(iv[i], f), (long long)ivf(oiv[i], f)); return; }
}

int main(int argc, char** argv) {
  if (argc > 1 && !strcmp(argv[1], "--constants")) {
    printf("DP_SMEM_ANCHORS=%u\n", DP_SMEM_ANCHORS);
    return 0;
  }
  char kind[8];
  while (scanf("%7s", kind) == 1) {
    if (kind[0] != 'D') return 2;
    int GL, NE, FB;
    unsigned band, c, nc;
    if (scanf("%d %d %d %u %u %u", &GL, &NE, &FB, &band, &c, &nc) != 6 || (GL != 4 && GL != 8)) return 2;
    std::vector<Chunk> chunks(nc);
    for (auto& C : chunks) {
      unsigned n;
      if (scanf("%u", &n) != 1) return 2;
      C.a.resize(n);
      for (unsigned t = 0; t < n; t++) {
        unsigned qc, qp, rcg, rp, rev;
        if (scanf("%u %u %u %u %u", &qc, &qp, &rcg, &rp, &rev) != 5) return 2;
        C.qctg = qc; C.a[t].qpos = qp; C.a[t].rpos = rp; C.a[t].rc = (rcg << 1) | rev;
      }
    }
    run_dp(GL, NE, FB != 0, band, c, chunks);
  }
  printf("dp configs %ld, chunks on chip %ld, chunks in global memory %ld, anchors %ld, intervals %ld, %d failures\n",
         n_dp_configs, n_chunks_onchip, n_chunks_global, n_anchors_all, n_iv_all, failures);
  return failures ? 1 : 0;
}
