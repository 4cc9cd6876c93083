// nj.cu -- sk_neighbor_joining and sk_neighbor_joining_multi: a neighbour-joining tree of a triangle's results on the GPU,
// on one context or with the distance matrix split over several.
//
// The edges come from cluster.cu's build_graph (its refusals apply unchanged).  They are scattered into a dense row-major
// float64 square over slots: 1.0 everywhere, 0 on the diagonal, 1 - ani for both directions of every edge.  Slots are in
// node-id order and stay so; a slot without a live node has R = NJ_DEAD.  On one context each step is two launches and no
// host round trip:
//   nj_scan_kernel    tiles of the upper triangle of the square (TILE x TILE, rows read 16 B per lane, R of the tile's rows
//                     and columns in shared memory), each thread keeps the (Q, i << 32 | j) minimum of its elements, a warp
//                     and block reduction gives the block's, and the last block to arrive reduces the blocks' minima and
//                     writes the chosen pair, its distance, R's, branch length and R_u to `sel`.  The order is total, so
//                     the result does not depend on scheduling.
//   nj_update_kernel  one thread per slot: row and column i become d_uk, R_k is updated, j is marked dead, and thread i
//                     writes join row t and renumbers its node.
// The host knows m = n - t at every step, so it sizes the grids and plans compactions without reading anything back: when
// m <= 3/4 of the square's dimension (and the square is more than one tile), the live slots are gathered in order into a
// square of dimension m.  The scan then reads at most (4/3)^2 of the live pairs.  The join table is read back once.
// Every formula is in nj_core.cuh, with each operation rounded on its own.
//
// On N > 1 contexts (nj_plan.hpp) context d holds the full rows of a band of slots [row0, row1), equal in row tiles; R and
// node are replicated and stay bit-identical, because every context computes them with the same formulas from the same
// inputs.  A step is three launches per context and two exchanges, ordered across contexts by events only (no kernel waits
// for another context):
//   nj_scan_kernel<true>  the context's planned tiles, a tile of another band's rows read transposed from its own rows (still
//                         evaluated as Q(i, j) with i < j and key i << 32 | j); the last block writes the context's
//                         (Q, key, d_ij) candidate.  The N candidates are copied to every context (24 B each).
//   nj_pick_kernel        every context reduces the N candidates in the same total order, so all pick the same join, and
//                         writes (d_ik, d_jk) of its band's rows k into the exchange vector; its band slice is copied to
//                         every other context (16 B per row).
//   nj_update_kernel      as on one context, with d_ik, d_jk from the exchange vector: it writes column i of the band's rows
//                         and, on i's owner, row i; context 0 writes the join table.
// A compaction reads the live slots back (once per compaction, O(log n) per tree) so that the host can size the row moves:
// each context gathers its band's live rows into a staging block, the new bands (of the compacted square) are filled from
// the staging blocks by peer copies, and the tiles are planned again.  Slot order is kept, so results do not change.
#include <cub/cub.cuh>
#include <thrust/iterator/counting_iterator.h>

#include <algorithm>
#include <chrono>
#include <cmath>
#include <string>
#include <vector>

#include "nj_core.cuh"
#include "nj_plan.hpp"
#include "sk_internal.h"
#include "store_ws.hpp"

using namespace sk;

namespace {

constexpr uint32_t TILE = 64;         // scan tile: TILE x TILE slots; the square's dimension is padded to a multiple
constexpr int SCAN_TPB = 256;         // 8 warps x 8 rows of a tile; a lane reads columns 2 lane, 2 lane + 1 of each row
constexpr int SCAN_BLOCKS_PER_SM = 4;
constexpr int TPB = 256;
constexpr uint32_t MAX_GENOMES = 1u << 24;   // 8 n^2 bytes is 2^51 here: far beyond any device
const char* const WHO = "sk_neighbor_joining";

struct NjBest {
  double q;
  uint64_t key;
};
struct NjCand {  // a context's minimum and its distance (several contexts)
  double q;
  uint64_t key;
  double dij;
};
struct NjSel {   // the step's join, as the scan's last block found it
  uint32_t i, j;
  double dij, di, ru;
};

inline uint32_t padded(uint32_t s) { return (s + TILE - 1) / TILE * TILE; }
inline unsigned blocks_for(uint64_t n) { return (unsigned)std::max<uint64_t>(1, (n + TPB - 1) / TPB); }

__device__ __forceinline__ void nj_take(double& q, uint64_t& k, double q2, uint64_t k2) {
  if (nj_before(q2, k2, q, k)) { q = q2; k = k2; }
}

// the block's minimum (q, k), valid in thread 0
__device__ void nj_block_min(double& q, uint64_t& k) {
  __shared__ double sq[32];
  __shared__ uint64_t sk[32];
  for (int o = 16; o; o >>= 1) nj_take(q, k, __shfl_down_sync(0xffffffffu, q, o), __shfl_down_sync(0xffffffffu, k, o));
  const int lane = threadIdx.x & 31, w = threadIdx.x >> 5, nw = blockDim.x >> 5;
  __syncthreads();   // sq / sk may still be read by an earlier call
  if (lane == 0) { sq[w] = q; sk[w] = k; }
  __syncthreads();
  if (w) return;
  q = lane < nw ? sq[lane] : INFINITY;
  k = lane < nw ? sk[lane] : UINT64_MAX;
  for (int o = 16; o; o >>= 1) nj_take(q, k, __shfl_down_sync(0xffffffffu, q, o), __shfl_down_sync(0xffffffffu, k, o));
}

// the N contexts' candidates reduced in context order (the order is total, so every context picks the same)
__device__ NjCand nj_pick(const NjCand* __restrict__ c, uint32_t N) {
  NjCand b = c[0];
  for (uint32_t d = 1; d < N; d++)
    if (nj_before(c[d].q, c[d].key, b.q, b.key)) b = c[d];
  return b;
}

// rows [row0, row0 + rows) of the square (dimension P), held from D: 1.0, diagonal 0 (padding included: its Q are +inf
// through R = NJ_DEAD, but stay finite)
__global__ void nj_fill_kernel(double* __restrict__ D, uint32_t P, uint32_t row0, uint32_t rows) {
  const uint64_t total = (uint64_t)rows * P;
  for (uint64_t x = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; x < total; x += (uint64_t)gridDim.x * blockDim.x)
    D[x] = row0 + x / P == x % P ? 0.0 : 1.0;
}

// both directions of every edge, where the row is in [row0, row1); the first row with ani > 1 goes to *bad (if given)
__global__ void nj_scatter_kernel(const uint64_t* __restrict__ ekey, const float* __restrict__ eani, const uint64_t* __restrict__ erow,
                                  uint64_t E, double* __restrict__ D, uint32_t P, uint32_t row0, uint32_t row1,
                                  unsigned long long* __restrict__ bad) {
  const uint64_t e = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (e >= E) return;
  const float ani = eani[e];
  if (bad && ani > 1.f) atomicMin(bad, (unsigned long long)erow[e]);
  const uint32_t a = (uint32_t)(ekey[e] >> 32), b = (uint32_t)ekey[e];
  const double d = nj_dist(ani);
  if (a >= row0 && a < row1) D[(size_t)(a - row0) * P + b] = d;
  if (b >= row0 && b < row1) D[(size_t)(b - row0) * P + a] = d;
}

// a warp per slot row0 + r, r < rows: R = the row sum over the n genomes (exact, so the order is free), NJ_DEAD for padding;
// node = the slot
__global__ void nj_rowsum_kernel(const double* __restrict__ D, uint32_t P, uint32_t n, uint32_t row0, uint32_t rows, double* __restrict__ R,
                                 uint32_t* __restrict__ node) {
  const uint32_t r = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
  if (r >= rows) return;
  const uint32_t g = row0 + r;
  double s = 0.0;
  if (g < n)
    for (uint32_t c = lane; c < n; c += 32) s = nj_add(s, D[(size_t)r * P + c]);
  for (int o = 16; o; o >>= 1) s = nj_add(s, __shfl_down_sync(0xffffffffu, s, o));
  if (lane == 0) { R[g] = g < n ? s : NJ_DEAD; node[g] = g; }
}

// The (Q, i, j) minimum over live pairs i < j of the square (m live nodes).  One context (BANDED = false): every tile of the
// upper triangle (nt tiles per side, n_tiles in all), and the last block to arrive writes the join to *sel.  Several
// (BANDED): the n_tiles tiles a << 32 | b of `tiles`, D holding the rows [row0, row1); a tile whose rows another context
// holds is read transposed from the rows of its columns.  The last block writes the context's candidate to *cand.  Either
// way the last block resets *arrived.
template <bool BANDED>
__global__ void __launch_bounds__(SCAN_TPB) nj_scan_kernel(const double* __restrict__ D, uint32_t P, const double* __restrict__ R, uint32_t m,
                                                           const uint64_t* __restrict__ tiles, uint64_t n_tiles, uint32_t row0, uint32_t row1,
                                                           NjBest* __restrict__ part, unsigned* __restrict__ arrived,
                                                           NjSel* __restrict__ sel, NjCand* __restrict__ cand) {
  __shared__ double rr[TILE], rc[TILE];
  __shared__ bool last;
  const uint32_t lane = threadIdx.x & 31, w = threadIdx.x >> 5;
  double bq = INFINITY;
  uint64_t bk = UINT64_MAX;
  for (uint64_t t = blockIdx.x; t < n_tiles; t += gridDim.x) {
    uint32_t r0, c0;
    if constexpr (BANDED) {
      const uint64_t x = tiles[t];
      r0 = (uint32_t)(x >> 32) * TILE;
      c0 = (uint32_t)x * TILE;
    } else {
      // tile t of the upper triangle, column by column: column tc holds the tiles (0..tc, tc)
      uint64_t tc = (uint64_t)((sqrt(8.0 * (double)t + 1.0) - 1.0) * 0.5);
      while (tc * (tc + 1) / 2 > t) tc--;
      while ((tc + 1) * (tc + 2) / 2 <= t) tc++;
      r0 = (uint32_t)(t - tc * (tc + 1) / 2) * TILE;
      c0 = (uint32_t)tc * TILE;
    }
    __syncthreads();
    if (threadIdx.x < TILE) rr[threadIdx.x] = R[r0 + threadIdx.x];
    else if (threadIdx.x < 2 * TILE) rc[threadIdx.x - TILE] = R[c0 + threadIdx.x - TILE];
    __syncthreads();
    if (!BANDED || (r0 >= row0 && r0 < row1)) {
      const uint32_t c = c0 + 2 * lane;
      const double rj0 = rc[2 * lane], rj1 = rc[2 * lane + 1];
      double2 v[8];
#pragma unroll
      for (int s = 0; s < 8; s++) v[s] = *(const double2*)(D + (size_t)(r0 - row0 + w + 8 * s) * P + c);
#pragma unroll
      for (int s = 0; s < 8; s++) {
        const uint32_t r = r0 + w + 8 * s;
        const double ri = rr[w + 8 * s];
        if (c > r) nj_take(bq, bk, nj_q(m, v[s].x, ri, rj0), (uint64_t)r << 32 | c);
        if (c + 1 > r) nj_take(bq, bk, nj_q(m, v[s].y, ri, rj1), (uint64_t)r << 32 | (c + 1));
      }
    } else {
      // transposed (r0 < c0: the tile is off the band's diagonal): row c of the square holds the tile's column c, and the
      // element (i, j) = D[j][i] has the bits of D[i][j]
      const uint32_t i = r0 + 2 * lane;
      const double ri0 = rr[2 * lane], ri1 = rr[2 * lane + 1];
      double2 v[8];
#pragma unroll
      for (int s = 0; s < 8; s++) v[s] = *(const double2*)(D + (size_t)(c0 - row0 + w + 8 * s) * P + i);
#pragma unroll
      for (int s = 0; s < 8; s++) {
        const uint32_t j = c0 + w + 8 * s;
        const double rj = rc[w + 8 * s];
        nj_take(bq, bk, nj_q(m, v[s].x, ri0, rj), (uint64_t)i << 32 | j);
        nj_take(bq, bk, nj_q(m, v[s].y, ri1, rj), (uint64_t)(i + 1) << 32 | j);
      }
    }
  }
  nj_block_min(bq, bk);
  if (threadIdx.x == 0) {
    part[blockIdx.x] = NjBest{bq, bk};
    __threadfence();
    last = atomicAdd(arrived, 1u) == gridDim.x - 1;
  }
  __syncthreads();
  if (!last) return;
  __threadfence();
  bq = INFINITY;
  bk = UINT64_MAX;
  for (uint32_t b = threadIdx.x; b < gridDim.x; b += blockDim.x)
    nj_take(bq, bk, __ldcg(&part[b].q), (uint64_t)__ldcg((const unsigned long long*)&part[b].key));
  nj_block_min(bq, bk);
  if (threadIdx.x == 0) {
    *arrived = 0;
    const uint32_t i = (uint32_t)(bk >> 32), j = (uint32_t)bk;
    if constexpr (BANDED) {   // no tiles: no candidate
      const double dij = bk == UINT64_MAX ? 0.0 : i >= row0 && i < row1 ? D[(size_t)(i - row0) * P + j] : D[(size_t)(j - row0) * P + i];
      *cand = NjCand{bq, bk, dij};
    } else {
      const double dij = D[(size_t)i * P + j], ri = R[i], rj = R[j];
      *sel = NjSel{i, j, dij, nj_delta_i(m, dij, ri, rj), nj_ru(m, ri, rj, dij)};
    }
  }
}

// several contexts: the join of the N candidates to *sel, and (d_ik, d_jk) of the band's rows row0 + k, k < rows, to xc
__global__ void nj_pick_kernel(const NjCand* __restrict__ cands, uint32_t N, const double* __restrict__ R, uint32_t m,
                               const double* __restrict__ D, uint32_t P, uint32_t row0, uint32_t rows, double2* __restrict__ xc,
                               NjSel* __restrict__ sel) {
  const NjCand b = nj_pick(cands, N);
  const uint32_t i = (uint32_t)(b.key >> 32), j = (uint32_t)b.key;
  const uint32_t k = blockIdx.x * blockDim.x + threadIdx.x;
  if (k == 0) {
    const double ri = R[i], rj = R[j];
    *sel = NjSel{i, j, b.dij, nj_delta_i(m, b.dij, ri, rj), nj_ru(m, ri, rj, b.dij)};
  }
  if (k < rows) xc[row0 + k] = make_double2(D[(size_t)k * P + i], D[(size_t)k * P + j]);
}

// join t (m live nodes before it): one thread per slot k < S.  D holds the rows [row0, row1); d_ik, d_jk come from rows i
// and j (xc == NULL: one context, which holds every row) or from the exchange vector xc.  joins may be NULL.
__global__ void nj_update_kernel(double* __restrict__ D, uint32_t P, uint32_t S, double* __restrict__ R, uint32_t* __restrict__ node,
                                 const NjSel* __restrict__ psel, uint32_t n, uint32_t t, sk_nj_join* __restrict__ joins, uint32_t row0,
                                 uint32_t row1, const double2* __restrict__ xc) {
  const uint32_t k = blockIdx.x * blockDim.x + threadIdx.x;
  if (k >= S) return;
  const NjSel s = *psel;
  if (k == s.j) { R[k] = NJ_DEAD; return; }
  if (k == s.i) {
    if (joins) joins[t] = sk_nj_join{node[s.i], node[s.j], s.di, nj_sub(s.dij, s.di)};
    node[k] = n + t;
    R[k] = s.ru;
    return;
  }
  const double rk = R[k];
  if (rk == NJ_DEAD) return;
  double dik, djk;
  if (xc) { const double2 x = xc[k]; dik = x.x; djk = x.y; }
  else { dik = D[(size_t)s.i * P + k]; djk = D[(size_t)s.j * P + k]; }
  const double duk = nj_duk(dik, djk, s.dij);
  if (s.i >= row0 && s.i < row1) D[(size_t)(s.i - row0) * P + k] = duk;
  if (k >= row0 && k < row1) D[(size_t)(k - row0) * P + s.i] = duk;
  R[k] = nj_rk(rk, dik, djk, duk);
}

// the last two live nodes, smaller id first, each at half their distance: found by a scan of R on one context, or (cands,
// several contexts) as the join of the candidates of a scan at m = 2, the only pair with a finite Q
__global__ void nj_last_kernel(const double* __restrict__ D, uint32_t P, uint32_t S, const double* __restrict__ R,
                               const uint32_t* __restrict__ node, uint32_t n, sk_nj_join* __restrict__ joins,
                               const NjCand* __restrict__ cands, uint32_t N) {
  uint32_t a = UINT32_MAX, b = UINT32_MAX;
  double d;
  if (cands) {
    const NjCand c = nj_pick(cands, N);
    a = (uint32_t)(c.key >> 32); b = (uint32_t)c.key; d = c.dij;
  } else {
    for (uint32_t k = 0; k < S && b == UINT32_MAX; k++)
      if (R[k] != NJ_DEAD) (a == UINT32_MAX ? a : b) = k;
    d = D[(size_t)a * P + b];
  }
  const double h = nj_mul(0.5, d);
  joins[n - 2] = sk_nj_join{node[a], node[b], h, h};
}

struct NjLive {
  const double* R;
  __device__ bool operator()(uint32_t k) const { return R[k] != NJ_DEAD; }
};

// compaction: rows [g0, g1) of the square of padded dimension P2 over the m live slots src[] (in order) of the square (P),
// whose rows from row0 on are held from D; row g goes to D2 + (g - g0) P2, padding as nj_fill_kernel
__global__ void nj_gather_kernel(const double* __restrict__ D, uint32_t P, uint32_t row0, const uint32_t* __restrict__ src, uint32_t m,
                                 uint32_t g0, uint32_t g1, double* __restrict__ D2, uint32_t P2) {
  const uint64_t total = (uint64_t)(g1 - g0) * P2;
  for (uint64_t x = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; x < total; x += (uint64_t)gridDim.x * blockDim.x) {
    const uint32_t r = g0 + (uint32_t)(x / P2), c = (uint32_t)(x % P2);
    D2[x] = r < m && c < m ? D[(size_t)(src[r] - row0) * P + src[c]] : r == c ? 0.0 : 1.0;
  }
}

__global__ void nj_gather_slots_kernel(const double* __restrict__ R, const uint32_t* __restrict__ node, const uint32_t* __restrict__ src,
                                       uint32_t m, uint32_t P2, double* __restrict__ R2, uint32_t* __restrict__ node2) {
  const uint32_t r = blockIdx.x * blockDim.x + threadIdx.x;
  if (r >= P2) return;
  R2[r] = r < m ? R[src[r]] : NJ_DEAD;
  node2[r] = r < m ? node[src[r]] : 0;
}

// one context's share: its rows [row0, row1) of the square (full rows, sq[cur]), the replicated R and node, its scan
// tiles (several contexts only) and the buffers of the step
struct Band {
  sk_ctx* c = nullptr;
  uint32_t row0 = 0, row1 = 0;
  DTmp<double> sq[2], R[2], stage;
  DTmp<uint32_t> node[2], src;
  DTmp<uint64_t> tiles, ekey;
  DTmp<float> eani;
  DTmp<unsigned long long> bad;
  DTmp<NjBest> part;
  DTmp<NjSel> sel;
  DTmp<NjCand> cands;
  DTmp<double2> xc;
  DTmp<unsigned> arrived;
  DTmp<int> n_sel;
  DTmp<uint8_t> tmp;
  uint64_t n_tiles = 0;
  cudaEvent_t ev[2] = {nullptr, nullptr};
  uint32_t rows() const { return row1 - row0; }
};

// every context's stream drained and its events destroyed when nj_impl returns, before the buffers go back to the arenas
// (a peer copy on one context's stream may read another context's buffer)
struct Drain {
  std::vector<Band>& b;
  ~Drain() {
    for (Band& x : b) {
      cudaSetDevice(x.c->device);
      cudaStreamSynchronize(x.c->stream);
      for (cudaEvent_t e : x.ev) if (e) cudaEventDestroy(e);
    }
    cudaGetLastError();
  }
};

int nj_impl(sk_ctx* const* ctxs, uint32_t N, uint32_t n, const sk_ani_result* results, uint64_t n_results, sk_nj_join* joins,
            sk_nj_stats* stats) {
  sk_ctx* const ctx0 = ctxs[0];
  std::vector<Band> B(N);
  for (uint32_t d = 0; d < N; d++) B[d].c = ctxs[d];
  Drain drain{B};
  // a failure of context d: its message on ctxs[0] as "context d: ..." (several contexts)
  const auto failed = [&](uint32_t d, int rc) {
    if (d) ctx0->err = "context " + std::to_string(d) + ": " + ctxs[d]->err;
    return rc;
  };
  // fn(ctx, band) on each context in turn, its device current
  const auto each = [&](auto fn) -> int {
    for (uint32_t d = 0; d < N; d++) {
      sk_ctx* ctx = ctxs[d];
      SK_CUDA(cudaSetDevice(ctx->device));
      const int rc = fn(ctx, B[d], d);
      if (rc != SK_OK) return failed(d, rc);
    }
    return SK_OK;
  };
  // ev[k] recorded on every context, then on every context the ranges [lo, hi) = range(d) of array(d) of every other context
  // d copied in (the waits also order a context's next writes after the others' reads of its range)
  const auto share = [&](int k, auto array, auto range) -> int {
    if (N == 1) return SK_OK;
    SK_TRY(each([&](sk_ctx* ctx, Band& b, uint32_t) -> int { SK_CUDA(cudaEventRecord(b.ev[k], ctx->stream)); return SK_OK; }));
    return each([&](sk_ctx* ctx, Band& b, uint32_t e) -> int {
      for (uint32_t d = 0; d < N; d++) {
        if (d == e) continue;
        SK_CUDA(cudaStreamWaitEvent(ctx->stream, B[d].ev[k], 0));
        const auto r = range(d);
        if (r.second > r.first)
          SK_CUDA(cudaMemcpyPeerAsync(array(b) + r.first, ctx->device, array(B[d]) + r.first, B[d].c->device,
                                      (r.second - r.first) * sizeof(*array(b)), ctx->stream));
      }
      return SK_OK;
    });
  };
  // every context's work so far ordered before every context's next work
  const auto barrier = [&]() { return share(1, [](Band& b) { return b.cands.p; }, [](uint32_t) { return std::make_pair((size_t)0, (size_t)0); }); };
  const auto launched = [](sk_ctx* ctx, unsigned k = 1) { count_launch(ctx, k); return cudaGetLastError(); };

  Graph g;
  {
    sk_ctx* ctx = ctx0;
    SK_CUDA(cudaSetDevice(ctx->device));
    SK_TRY(build_graph(ctx, WHO, n, results, n_results, 0.f, g));
  }
  const uint64_t E = g.E;
  for (int b = 0; b < 2; b++) { g.key[b].release(); g.val[b].release(); }   // the CSR is not needed
  g.off.release();
  if (stats) { stats->n_edges = E; stats->joins = 0; stats->compactions = 0; }
  if (N > 1) {
    enable_peer_access(ctxs, N);
    SK_TRY(each([&](sk_ctx* ctx, Band& b, uint32_t) -> int {
      for (cudaEvent_t& e : b.ev) SK_CUDA(cudaEventCreateWithFlags(&e, cudaEventDisableTiming));
      return SK_OK;
    }));
  }
  // the bands of a square of dimension P, and (several contexts) their scan tiles
  const auto plan = [&](uint32_t P, std::vector<std::vector<uint64_t>>* tiles) {
    const std::vector<uint32_t> band = sknj::nj_bands(P / TILE, N);
    for (uint32_t d = 0; d < N; d++) { B[d].row0 = band[d] * TILE; B[d].row1 = band[d + 1] * TILE; }
    if (tiles) *tiles = sknj::plan_nj(P / TILE, N).tiles;
  };
  // the first compaction gathers floor(3n / 4) slots (only when the square is more than one tile)
  const uint32_t first_m = n > TILE ? (uint32_t)(3ull * n / 4) : 0;
  uint32_t S = n, P = padded(n);
  double need = 0;   // per context: its rows of the square and of the first compaction's square
  if (n <= MAX_GENOMES) {
    const uint32_t P1 = padded(first_m);
    const std::vector<uint32_t> b0 = sknj::nj_bands(P / TILE, N), b1 = sknj::nj_bands(P1 / TILE, N);
    for (uint32_t d = 0; d < N; d++)
      need = std::max(need, 8.0 * TILE * (b0[d + 1] - b0[d]) * P + 8.0 * TILE * (b1[d + 1] - b1[d]) * P1);
  }
  const auto nomem = [&](uint32_t d) {
    cudaGetLastError();
    char b[64];
    snprintf(b, sizeof(b), "%.0f", n > MAX_GENOMES ? 8.0 * (double)n * n / N : need);
    ctxs[d]->err = std::string(WHO) + ": out of device memory: the distance matrix of " + std::to_string(n) + " genomes and its first compaction need " +
                   b + " bytes" + (N > 1 ? " per context on " + std::to_string(N) + " contexts" : "");
    return failed(d, SK_ERR_NOMEM);
  };
  if (n > MAX_GENOMES) return nomem(0);
  std::vector<std::vector<uint64_t>> tiles;
  plan(P, N > 1 ? &tiles : nullptr);
  for (uint32_t d = 0; n >= 2 && d < N; d++) {
    sk_ctx* ctx = ctxs[d];
    SK_CUDA(cudaSetDevice(ctx->device));
    if (B[d].sq[0].alloc((uint64_t)B[d].rows() * P, ctx) != cudaSuccess) return nomem(d);
    if (N == 1 && first_m && B[d].sq[1].alloc((uint64_t)padded(first_m) * padded(first_m), ctx) != cudaSuccess) return nomem(d);
  }
  {
    sk_ctx* ctx = ctx0;
    SK_TRY(cl_alloc(ctx, B[0].bad, 1, "bad row", WHO));
    SK_CUDA(cudaMemsetAsync(B[0].bad.p, 0xff, 8, ctx->stream));
  }
  if (N > 1 && E) {   // the edges on every context
    {
      sk_ctx* ctx = ctx0;
      SK_CUDA(cudaEventRecord(B[0].ev[0], ctx->stream));
    }
    SK_TRY(each([&](sk_ctx* ctx, Band& b, uint32_t d) -> int {
      if (d == 0) return SK_OK;
      SK_TRY(cl_alloc(ctx, b.ekey, E, "edge keys", WHO));
      SK_TRY(cl_alloc(ctx, b.eani, E, "edge ANIs", WHO));
      SK_CUDA(cudaStreamWaitEvent(ctx->stream, B[0].ev[0], 0));
      SK_CUDA(cudaMemcpyPeerAsync(b.ekey.p, ctx->device, g.ekey.p, ctx0->device, E * 8, ctx->stream));
      SK_CUDA(cudaMemcpyPeerAsync(b.eani.p, ctx->device, g.eani.p, ctx0->device, E * 4, ctx->stream));
      return SK_OK;
    }));
  }
  SK_TRY(each([&](sk_ctx* ctx, Band& b, uint32_t d) -> int {
    cudaStream_t st = ctx->stream;
    if (n >= 2 && b.rows()) {
      nj_fill_kernel<<<ctx->sm_count * 8, TPB, 0, st>>>(b.sq[0].p, P, b.row0, b.rows());
      SK_CUDA(launched(ctx));
    }
    if (E && (b.rows() != 0 || d == 0)) {   // context 0 checks every edge (its band may be empty)
      nj_scatter_kernel<<<blocks_for(E), TPB, 0, st>>>(d ? b.ekey.p : g.ekey.p, d ? b.eani.p : g.eani.p, g.erow.p, E, n >= 2 ? b.sq[0].p : nullptr,
                                                       P, b.row0, n >= 2 ? b.row1 : 0, d ? nullptr : b.bad.p);
      SK_CUDA(launched(ctx));
    }
    return SK_OK;
  }));
  {
    sk_ctx* ctx = ctx0;
    cudaStream_t st = ctx->stream;
    unsigned long long h_bad = 0;
    SK_CUDA(cudaSetDevice(ctx->device));
    SK_CUDA(cudaMemcpyAsync(&h_bad, B[0].bad.p, 8, cudaMemcpyDeviceToHost, st));
    SK_CUDA(cudaStreamSynchronize(st));
    if (h_bad != UINT64_MAX) { ctx->err = std::string(WHO) + ": ani > 1 (a negative distance) in " + row_text(results, h_bad); return SK_ERR_PARAM; }
  }
  if (n < 2) return SK_OK;
  SK_TRY(each([&](sk_ctx* ctx, Band& b, uint32_t) -> int {   // after the scatter, in stream order
    b.ekey.release(); b.eani.release();
    return SK_OK;
  }));
  if (N > 1) SK_TRY(barrier());   // the other contexts' copies read ctxs[0]'s edges
  g.ekey.release(); g.eani.release(); g.erow.release();
  DTmp<sk_nj_join> d_joins;
  const thrust::counting_iterator<uint32_t> idx(0);
  size_t tb = 0;
  SK_TRY(each([&](sk_ctx* ctx, Band& b, uint32_t d) -> int {
    cudaStream_t st = ctx->stream;
    const unsigned scan_cap = (unsigned)ctx->sm_count * SCAN_BLOCKS_PER_SM;
    for (int k = 0; k < 2; k++) {
      SK_TRY(cl_alloc(ctx, b.R[k], P, "row sums", WHO));
      SK_TRY(cl_alloc(ctx, b.node[k], P, "node numbers", WHO));
    }
    SK_TRY(cl_alloc(ctx, b.src, P, "live slots", WHO));
    SK_TRY(cl_alloc(ctx, b.part, scan_cap, "block minima", WHO));
    SK_TRY(cl_alloc(ctx, b.sel, 1, "join", WHO));
    SK_TRY(cl_alloc(ctx, b.arrived, 1, "arrival counter", WHO));
    if (d == 0) SK_TRY(cl_alloc(ctx, d_joins, n - 1, "join table", WHO));
    SK_TRY(cl_alloc(ctx, b.n_sel, 1, "live count", WHO));
    if (N > 1) {
      SK_TRY(cl_alloc(ctx, b.cands, N, "context minima", WHO));
      SK_TRY(cl_alloc(ctx, b.xc, P, "exchanged columns", WHO));
      SK_TRY(cl_alloc(ctx, b.tiles, tiles[d].size(), "scan tiles", WHO));
      if (!tiles[d].empty()) SK_CUDA(cudaMemcpyAsync(b.tiles.p, tiles[d].data(), tiles[d].size() * 8, cudaMemcpyHostToDevice, st));
      b.n_tiles = tiles[d].size();
    }
    SK_CUDA(cudaMemsetAsync(b.arrived.p, 0, 4, st));
    if (b.rows()) {
      nj_rowsum_kernel<<<(unsigned)(((uint64_t)b.rows() * 32 + TPB - 1) / TPB), TPB, 0, st>>>(b.sq[0].p, P, n, b.row0, b.rows(), b.R[0].p, b.node[0].p);
      SK_CUDA(launched(ctx));
    }
    SK_CUDA(cub::DeviceSelect::If(nullptr, tb, idx, b.src.p, b.n_sel.p, (int)n, NjLive{b.R[0].p}, st));
    SK_TRY(cl_alloc(ctx, b.tmp, tb, "select temporaries", WHO));
    return SK_OK;
  }));
  const auto band_rows = [&](uint32_t d) { return std::make_pair((size_t)B[d].row0, (size_t)B[d].row1); };
  SK_TRY(share(0, [](Band& b) { return b.R[0].p; }, band_rows));
  SK_TRY(share(1, [](Band& b) { return b.node[0].p; }, band_rows));
  int cur = 0;
  uint32_t compactions = 0;
  std::vector<uint32_t> h_src;
  // the m live slots gathered, in order, into a square of dimension m
  const auto compact = [&](uint32_t m) -> int {
    const uint32_t P2 = padded(m);
    std::vector<std::pair<uint32_t, uint32_t>> live(N, {0, P2});   // rows of the new square each context gathers
    SK_TRY(each([&](sk_ctx* ctx, Band& b, uint32_t) -> int {
      SK_CUDA(cub::DeviceSelect::If(b.tmp.p, tb, idx, b.src.p, b.n_sel.p, (int)S, NjLive{b.R[cur].p}, ctx->stream));
      return SK_OK;
    }));
    if (N > 1) {   // the live rows of each band: the host sizes the moves
      sk_ctx* ctx = ctx0;
      h_src.resize(m);
      SK_CUDA(cudaSetDevice(ctx->device));
      SK_CUDA(cudaMemcpyAsync(h_src.data(), B[0].src.p, (size_t)m * 4, cudaMemcpyDeviceToHost, ctx->stream));
      SK_CUDA(cudaStreamSynchronize(ctx->stream));
      for (uint32_t d = 0; d < N; d++)
        live[d] = {(uint32_t)(std::lower_bound(h_src.begin(), h_src.end(), B[d].row0) - h_src.begin()),
                   (uint32_t)(std::lower_bound(h_src.begin(), h_src.end(), B[d].row1) - h_src.begin())};
    }
    SK_TRY(each([&](sk_ctx* ctx, Band& b, uint32_t d) -> int {
      cudaStream_t st = ctx->stream;
      const uint32_t g0 = live[d].first, g1 = live[d].second;
      DTmp<double>& to = N == 1 ? b.sq[cur ^ 1] : b.stage;   // one context gathers straight into the new square
      const uint64_t count = (uint64_t)(g1 - g0) * P2;
      if (to.n < count && cl_alloc(ctx, to, count, N == 1 ? "compacted distance matrix" : "compaction staging", WHO) != SK_OK) return SK_ERR_NOMEM;
      if (g1 > g0) nj_gather_kernel<<<ctx->sm_count * 8, TPB, 0, st>>>(b.sq[cur].p, P, b.row0, b.src.p, m, g0, g1, to.p, P2);
      nj_gather_slots_kernel<<<blocks_for(P2), TPB, 0, st>>>(b.R[cur].p, b.node[cur].p, b.src.p, m, P2, b.R[cur ^ 1].p, b.node[cur ^ 1].p);
      SK_CUDA(launched(ctx, g1 > g0 ? 3 : 2));
      b.sq[cur].release();
      return SK_OK;
    }));
    if (N > 1) {   // the new bands, filled from the staging blocks
      const std::vector<uint32_t> old0 = [&] { std::vector<uint32_t> v(N); for (uint32_t d = 0; d < N; d++) v[d] = live[d].first; return v; }();
      SK_TRY(each([&](sk_ctx* ctx, Band& b, uint32_t) -> int { SK_CUDA(cudaEventRecord(b.ev[0], ctx->stream)); return SK_OK; }));
      plan(P2, &tiles);
      SK_TRY(each([&](sk_ctx* ctx, Band& b, uint32_t e) -> int {
        cudaStream_t st = ctx->stream;
        if (cl_alloc(ctx, b.sq[cur ^ 1], (uint64_t)b.rows() * P2, "compacted distance matrix", WHO) != SK_OK) return SK_ERR_NOMEM;
        for (uint32_t d = 0; d < N; d++) {
          SK_CUDA(cudaStreamWaitEvent(st, B[d].ev[0], 0));
          const uint32_t lo = std::max(live[d].first, b.row0), hi = std::min(live[d].second, b.row1);
          if (hi > lo)
            SK_CUDA(cudaMemcpyPeerAsync(b.sq[cur ^ 1].p + (size_t)(lo - b.row0) * P2, ctx->device, B[d].stage.p + (size_t)(lo - old0[d]) * P2,
                                        B[d].c->device, (size_t)(hi - lo) * P2 * 8, st));
        }
        const uint32_t p0 = std::max(m, b.row0);   // padding rows
        if (b.row1 > p0) {
          nj_gather_kernel<<<ctx->sm_count * 8, TPB, 0, st>>>(nullptr, 0, 0, nullptr, m, p0, b.row1, b.sq[cur ^ 1].p + (size_t)(p0 - b.row0) * P2, P2);
          SK_CUDA(launched(ctx));
        }
        if (b.tiles.n < tiles[e].size()) SK_TRY(cl_alloc(ctx, b.tiles, tiles[e].size(), "scan tiles", WHO));
        if (!tiles[e].empty()) SK_CUDA(cudaMemcpyAsync(b.tiles.p, tiles[e].data(), tiles[e].size() * 8, cudaMemcpyHostToDevice, st));
        b.n_tiles = tiles[e].size();
        SK_CUDA(cudaEventRecord(b.ev[1], st));
        return SK_OK;
      }));
      SK_TRY(each([&](sk_ctx* ctx, Band& b, uint32_t) -> int {   // every staging block copied: it may go
        for (uint32_t d = 0; d < N; d++) SK_CUDA(cudaStreamWaitEvent(ctx->stream, B[d].ev[1], 0));
        b.stage.release();
        return SK_OK;
      }));
    }
    cur ^= 1;
    S = m;
    P = P2;
    compactions++;
    return SK_OK;
  };
  // the step's scan (several contexts: and the exchange of the candidates) for m live nodes
  const auto scan = [&](uint32_t m) -> int {
    SK_TRY(each([&](sk_ctx* ctx, Band& b, uint32_t d) -> int {
      const unsigned scan_cap = (unsigned)ctx->sm_count * SCAN_BLOCKS_PER_SM;
      if (N == 1) {
        const uint64_t nt = P / TILE, n_tiles = nt * (nt + 1) / 2;
        nj_scan_kernel<false><<<(unsigned)std::min<uint64_t>(n_tiles, scan_cap), SCAN_TPB, 0, ctx->stream>>>(
            b.sq[cur].p, P, b.R[cur].p, m, nullptr, n_tiles, 0, P, b.part.p, b.arrived.p, b.sel.p, nullptr);
      } else {
        nj_scan_kernel<true><<<(unsigned)std::max<uint64_t>(1, std::min<uint64_t>(b.n_tiles, scan_cap)), SCAN_TPB, 0, ctx->stream>>>(
            b.sq[cur].p, P, b.R[cur].p, m, b.tiles.p, b.n_tiles, b.row0, b.row1, b.part.p, b.arrived.p, nullptr, b.cands.p + d);
      }
      SK_CUDA(launched(ctx));
      return SK_OK;
    }));
    return share(0, [](Band& b) { return b.cands.p; }, [](uint32_t d) { return std::make_pair((size_t)d, (size_t)d + 1); });
  };
  for (uint32_t t = 0; t + 2 < n; t++) {
    const uint32_t m = n - t;
    if (S > TILE && 4ull * m <= 3ull * S) SK_TRY(compact(m));
    SK_TRY(scan(m));
    if (N > 1) {
      SK_TRY(each([&](sk_ctx* ctx, Band& b, uint32_t) -> int {
        const uint32_t rows = b.row0 < S ? std::min(b.row1, S) - b.row0 : 0;
        nj_pick_kernel<<<blocks_for(rows), TPB, 0, ctx->stream>>>(b.cands.p, N, b.R[cur].p, m, b.sq[cur].p, P, b.row0, rows, b.xc.p, b.sel.p);
        SK_CUDA(launched(ctx));
        return SK_OK;
      }));
      SK_TRY(share(1, [](Band& b) { return b.xc.p; }, [&](uint32_t d) {
        return std::make_pair((size_t)std::min(B[d].row0, S), (size_t)std::min(B[d].row1, S));
      }));
    }
    SK_TRY(each([&](sk_ctx* ctx, Band& b, uint32_t d) -> int {
      nj_update_kernel<<<blocks_for(S), TPB, 0, ctx->stream>>>(b.sq[cur].p, P, S, b.R[cur].p, b.node[cur].p, b.sel.p, n, t,
                                                                d ? nullptr : d_joins.p, b.row0, b.row1, N > 1 ? b.xc.p : nullptr);
      SK_CUDA(launched(ctx));
      return SK_OK;
    }));
  }
  if (N > 1) SK_TRY(scan(2));
  {
    sk_ctx* ctx = ctx0;
    cudaStream_t st = ctx->stream;
    SK_CUDA(cudaSetDevice(ctx->device));
    nj_last_kernel<<<1, 1, 0, st>>>(B[0].sq[cur].p, P, S, B[0].R[cur].p, B[0].node[cur].p, n, d_joins.p, N > 1 ? B[0].cands.p : nullptr, N);
    SK_CUDA(launched(ctx));
    SK_CUDA(cudaMemcpyAsync(joins, d_joins.p, (size_t)(n - 1) * sizeof(sk_nj_join), cudaMemcpyDeviceToHost, st));
    SK_CUDA(cudaStreamSynchronize(st));
  }
  if (stats) { stats->joins = n - 1; stats->compactions = compactions; }
  return SK_OK;
}

int nj_entry(sk_ctx* const* ctxs, uint32_t n_ctx, uint32_t n_genomes, const sk_ani_result* results, uint64_t n_results, sk_nj_join* joins,
             sk_nj_stats* stats) {
  sk_ctx* ctx = ctxs[0];
  if ((n_results && !results) || (n_genomes > 1 && !joins)) { ctx->err = std::string(WHO) + ": NULL argument"; return SK_ERR_PARAM; }
  SK_CUDA(cudaSetDevice(ctx->device));
  const auto t0 = std::chrono::steady_clock::now();
  const int rc = nj_impl(ctxs, n_ctx, n_genomes, results, n_results, joins, stats);
  cudaSetDevice(ctx->device);
  if (rc == SK_OK && stats) stats->t_device = std::chrono::duration<double>(std::chrono::steady_clock::now() - t0).count();
  return rc;
}

}  // namespace

int sk_neighbor_joining(sk_ctx* ctx, uint32_t n_genomes, const sk_ani_result* results, uint64_t n_results, sk_nj_join* joins,
                        sk_nj_stats* stats) {
  if (!ctx) return SK_ERR_PARAM;
  return nj_entry(&ctx, 1, n_genomes, results, n_results, joins, stats);
}

int sk_neighbor_joining_multi(sk_ctx* const* ctxs, uint32_t n_ctx, uint32_t n_genomes, const sk_ani_result* results, uint64_t n_results,
                              sk_nj_join* joins, sk_nj_stats* stats) {
  if (!ctxs || !n_ctx || !ctxs[0]) return SK_ERR_PARAM;
  SK_TRY(check_contexts(ctxs, n_ctx));
  return nj_entry(ctxs, n_ctx, n_genomes, results, n_results, joins, stats);
}
