// nj.cu -- sk_neighbor_joining: a neighbour-joining tree of a triangle's results on the GPU.
//
// The edges come from cluster.cu's build_graph (its refusals apply unchanged).  They are scattered into a dense row-major
// float64 square over slots: 1.0 everywhere, 0 on the diagonal, 1 - ani for both directions of every edge.  Slots are in
// node-id order and stay so; a slot without a live node has R = NJ_DEAD.  Each step is two launches and no host round trip:
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
#include <cub/cub.cuh>
#include <thrust/iterator/counting_iterator.h>

#include <algorithm>
#include <chrono>
#include <cmath>
#include <string>

#include "nj_core.cuh"
#include "sk_internal.h"

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

// D = 1.0, diagonal 0 (padding included: its Q are +inf through R = NJ_DEAD, but stay finite)
__global__ void nj_fill_kernel(double* __restrict__ D, uint32_t P) {
  const uint64_t total = (uint64_t)P * P;
  for (uint64_t x = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; x < total; x += (uint64_t)gridDim.x * blockDim.x)
    D[x] = x / P == x % P ? 0.0 : 1.0;
}

// both directions of every edge; the first row with ani > 1 goes to *bad
__global__ void nj_scatter_kernel(const uint64_t* __restrict__ ekey, const float* __restrict__ eani, const uint64_t* __restrict__ erow,
                                  uint64_t E, double* __restrict__ D, uint32_t P, unsigned long long* __restrict__ bad) {
  const uint64_t e = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (e >= E) return;
  const float ani = eani[e];
  if (ani > 1.f) atomicMin(bad, (unsigned long long)erow[e]);
  const uint32_t a = (uint32_t)(ekey[e] >> 32), b = (uint32_t)ekey[e];
  const double d = nj_dist(ani);
  D[(size_t)a * P + b] = d;
  D[(size_t)b * P + a] = d;
}

// a warp per slot: R = the row sum over the n genomes (exact, so the order is free), NJ_DEAD for padding; node = the slot
__global__ void nj_rowsum_kernel(const double* __restrict__ D, uint32_t P, uint32_t n, double* __restrict__ R, uint32_t* __restrict__ node) {
  const uint32_t r = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
  if (r >= P) return;
  double s = 0.0;
  if (r < n)
    for (uint32_t c = lane; c < n; c += 32) s = nj_add(s, D[(size_t)r * P + c]);
  for (int o = 16; o; o >>= 1) s = nj_add(s, __shfl_down_sync(0xffffffffu, s, o));
  if (lane == 0) { R[r] = r < n ? s : NJ_DEAD; node[r] = r; }
}

// the (Q, i, j) minimum over live pairs i < j of the square (m live nodes, nt tiles per side); the last block to arrive
// writes the join to *sel and resets *arrived
__global__ void __launch_bounds__(SCAN_TPB) nj_scan_kernel(const double* __restrict__ D, uint32_t P, const double* __restrict__ R, uint32_t m,
                                                           uint64_t n_tiles, NjBest* __restrict__ part, unsigned* __restrict__ arrived,
                                                           NjSel* __restrict__ sel) {
  __shared__ double rr[TILE], rc[TILE];
  __shared__ bool last;
  const uint32_t lane = threadIdx.x & 31, w = threadIdx.x >> 5;
  double bq = INFINITY;
  uint64_t bk = UINT64_MAX;
  for (uint64_t t = blockIdx.x; t < n_tiles; t += gridDim.x) {
    // tile t of the upper triangle, column by column: column tc holds the tiles (0..tc, tc)
    uint64_t tc = (uint64_t)((sqrt(8.0 * (double)t + 1.0) - 1.0) * 0.5);
    while (tc * (tc + 1) / 2 > t) tc--;
    while ((tc + 1) * (tc + 2) / 2 <= t) tc++;
    const uint32_t r0 = (uint32_t)(t - tc * (tc + 1) / 2) * TILE, c0 = (uint32_t)tc * TILE;
    __syncthreads();
    if (threadIdx.x < TILE) rr[threadIdx.x] = R[r0 + threadIdx.x];
    else if (threadIdx.x < 2 * TILE) rc[threadIdx.x - TILE] = R[c0 + threadIdx.x - TILE];
    __syncthreads();
    const uint32_t c = c0 + 2 * lane;
    const double rj0 = rc[2 * lane], rj1 = rc[2 * lane + 1];
    double2 v[8];
#pragma unroll
    for (int s = 0; s < 8; s++) v[s] = *(const double2*)(D + (size_t)(r0 + w + 8 * s) * P + c);
#pragma unroll
    for (int s = 0; s < 8; s++) {
      const uint32_t r = r0 + w + 8 * s;
      const double ri = rr[w + 8 * s];
      if (c > r) nj_take(bq, bk, nj_q(m, v[s].x, ri, rj0), (uint64_t)r << 32 | c);
      if (c + 1 > r) nj_take(bq, bk, nj_q(m, v[s].y, ri, rj1), (uint64_t)r << 32 | (c + 1));
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
    const double dij = D[(size_t)i * P + j], ri = R[i], rj = R[j];
    *sel = NjSel{i, j, dij, nj_delta_i(m, dij, ri, rj), nj_ru(m, ri, rj, dij)};
  }
}

// join t (m live nodes before it): one thread per slot k < S
__global__ void nj_update_kernel(double* __restrict__ D, uint32_t P, uint32_t S, double* __restrict__ R, uint32_t* __restrict__ node,
                                 const NjSel* __restrict__ psel, uint32_t n, uint32_t t, sk_nj_join* __restrict__ joins) {
  const uint32_t k = blockIdx.x * blockDim.x + threadIdx.x;
  if (k >= S) return;
  const NjSel s = *psel;
  if (k == s.j) { R[k] = NJ_DEAD; return; }
  if (k == s.i) {
    joins[t] = sk_nj_join{node[s.i], node[s.j], s.di, nj_sub(s.dij, s.di)};
    node[k] = n + t;
    R[k] = s.ru;
    return;
  }
  const double rk = R[k];
  if (rk == NJ_DEAD) return;
  const double dik = D[(size_t)s.i * P + k], djk = D[(size_t)s.j * P + k];
  const double duk = nj_duk(dik, djk, s.dij);
  D[(size_t)s.i * P + k] = duk;
  D[(size_t)k * P + s.i] = duk;
  R[k] = nj_rk(rk, dik, djk, duk);
}

// the last two live nodes, smaller id first, each at half their distance
__global__ void nj_last_kernel(const double* __restrict__ D, uint32_t P, uint32_t S, const double* __restrict__ R,
                               const uint32_t* __restrict__ node, uint32_t n, sk_nj_join* __restrict__ joins) {
  uint32_t a = UINT32_MAX, b = UINT32_MAX;
  for (uint32_t k = 0; k < S && b == UINT32_MAX; k++)
    if (R[k] != NJ_DEAD) (a == UINT32_MAX ? a : b) = k;
  const double h = nj_mul(0.5, D[(size_t)a * P + b]);
  joins[n - 2] = sk_nj_join{node[a], node[b], h, h};
}

struct NjLive {
  const double* R;
  __device__ bool operator()(uint32_t k) const { return R[k] != NJ_DEAD; }
};

// compaction: the m live slots src[] (in order) of the square (P) -> a square of padded dimension P2, padding as nj_fill_kernel
__global__ void nj_gather_kernel(const double* __restrict__ D, uint32_t P, const uint32_t* __restrict__ src, uint32_t m,
                                 double* __restrict__ D2, uint32_t P2) {
  const uint64_t total = (uint64_t)P2 * P2;
  for (uint64_t x = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; x < total; x += (uint64_t)gridDim.x * blockDim.x) {
    const uint32_t r = (uint32_t)(x / P2), c = (uint32_t)(x % P2);
    D2[x] = r < m && c < m ? D[(size_t)src[r] * P + src[c]] : r == c ? 0.0 : 1.0;
  }
}

__global__ void nj_gather_slots_kernel(const double* __restrict__ R, const uint32_t* __restrict__ node, const uint32_t* __restrict__ src,
                                       uint32_t m, uint32_t P2, double* __restrict__ R2, uint32_t* __restrict__ node2) {
  const uint32_t r = blockIdx.x * blockDim.x + threadIdx.x;
  if (r >= P2) return;
  R2[r] = r < m ? R[src[r]] : NJ_DEAD;
  node2[r] = r < m ? node[src[r]] : 0;
}

int nj_impl(sk_ctx* ctx, uint32_t n, const sk_ani_result* results, uint64_t n_results, sk_nj_join* joins, sk_nj_stats* stats) {
  cudaStream_t st = ctx->stream;
  const auto launched = [&](unsigned k = 1) { count_launch(ctx, k); return cudaGetLastError(); };
  Graph g;
  SK_TRY(build_graph(ctx, WHO, n, results, n_results, 0.f, g));
  const uint64_t E = g.E;
  for (int b = 0; b < 2; b++) { g.key[b].release(); g.val[b].release(); }   // the CSR is not needed
  g.off.release();
  if (stats) { stats->n_edges = E; stats->joins = 0; stats->compactions = 0; }
  // the first compaction gathers floor(3n / 4) slots (only when the square is more than one tile)
  const uint32_t first_m = n > TILE ? (uint32_t)(3ull * n / 4) : 0;
  const double need = 8.0 * (double)padded(std::min(n, MAX_GENOMES)) * padded(std::min(n, MAX_GENOMES)) +
                      8.0 * (double)padded(first_m) * padded(first_m);
  const auto nomem = [&]() {
    cudaGetLastError();
    char b[64];
    snprintf(b, sizeof(b), "%.0f", n > MAX_GENOMES ? 8.0 * (double)n * n : need);
    ctx->err = std::string(WHO) + ": out of device memory: the distance matrix of " + std::to_string(n) + " genomes and its first compaction need " +
               b + " bytes";
    return SK_ERR_NOMEM;
  };
  if (n > MAX_GENOMES) return nomem();
  uint32_t S = n, P = padded(n);
  DTmp<double> sq[2], R[2];
  DTmp<uint32_t> node[2], src;
  DTmp<unsigned long long> bad;
  if (n >= 2) {
    if (sq[0].alloc((uint64_t)P * P, ctx) != cudaSuccess) return nomem();
    if (first_m && sq[1].alloc((uint64_t)padded(first_m) * padded(first_m), ctx) != cudaSuccess) return nomem();
  }
  SK_TRY(cl_alloc(ctx, bad, 1, "bad row", WHO));
  SK_CUDA(cudaMemsetAsync(bad.p, 0xff, 8, st));
  if (n >= 2) {
    nj_fill_kernel<<<ctx->sm_count * 8, TPB, 0, st>>>(sq[0].p, P);
    SK_CUDA(launched());
  }
  if (E) {
    nj_scatter_kernel<<<blocks_for(E), TPB, 0, st>>>(g.ekey.p, g.eani.p, g.erow.p, E, n >= 2 ? sq[0].p : nullptr, P, bad.p);
    SK_CUDA(launched());
  }
  unsigned long long h_bad = 0;
  SK_CUDA(cudaMemcpyAsync(&h_bad, bad.p, 8, cudaMemcpyDeviceToHost, st));
  SK_CUDA(cudaStreamSynchronize(st));
  if (h_bad != UINT64_MAX) { ctx->err = std::string(WHO) + ": ani > 1 (a negative distance) in " + row_text(results, h_bad); return SK_ERR_PARAM; }
  if (n < 2) return SK_OK;
  g.ekey.release(); g.eani.release(); g.erow.release();
  const unsigned scan_cap = (unsigned)ctx->sm_count * SCAN_BLOCKS_PER_SM;
  DTmp<NjBest> part;
  DTmp<NjSel> sel;
  DTmp<unsigned> arrived;
  DTmp<sk_nj_join> d_joins;
  DTmp<int> n_sel;
  for (int b = 0; b < 2; b++) {
    SK_TRY(cl_alloc(ctx, R[b], P, "row sums", WHO));
    SK_TRY(cl_alloc(ctx, node[b], P, "node numbers", WHO));
  }
  SK_TRY(cl_alloc(ctx, src, P, "live slots", WHO));
  SK_TRY(cl_alloc(ctx, part, scan_cap, "block minima", WHO));
  SK_TRY(cl_alloc(ctx, sel, 1, "join", WHO));
  SK_TRY(cl_alloc(ctx, arrived, 1, "arrival counter", WHO));
  SK_TRY(cl_alloc(ctx, d_joins, n - 1, "join table", WHO));
  SK_TRY(cl_alloc(ctx, n_sel, 1, "live count", WHO));
  SK_CUDA(cudaMemsetAsync(arrived.p, 0, 4, st));
  nj_rowsum_kernel<<<(unsigned)(((uint64_t)P * 32 + TPB - 1) / TPB), TPB, 0, st>>>(sq[0].p, P, n, R[0].p, node[0].p);
  SK_CUDA(launched());
  size_t tb = 0;
  const thrust::counting_iterator<uint32_t> idx(0);
  SK_CUDA(cub::DeviceSelect::If(nullptr, tb, idx, src.p, n_sel.p, (int)n, NjLive{R[0].p}, st));
  DTmp<uint8_t> tmp;
  SK_TRY(cl_alloc(ctx, tmp, tb, "select temporaries", WHO));
  int cur = 0;
  uint32_t compactions = 0;
  for (uint32_t t = 0; t + 2 < n; t++) {
    const uint32_t m = n - t;
    if (S > TILE && 4ull * m <= 3ull * S) {   // gather the m live slots, in order, into a square of dimension m
      const uint32_t P2 = padded(m);
      if (sq[cur ^ 1].n < (uint64_t)P2 * P2 && cl_alloc(ctx, sq[cur ^ 1], (uint64_t)P2 * P2, "compacted distance matrix", WHO) != SK_OK)
        return SK_ERR_NOMEM;
      SK_CUDA(cub::DeviceSelect::If(tmp.p, tb, idx, src.p, n_sel.p, (int)S, NjLive{R[cur].p}, st));
      nj_gather_kernel<<<ctx->sm_count * 8, TPB, 0, st>>>(sq[cur].p, P, src.p, m, sq[cur ^ 1].p, P2);
      nj_gather_slots_kernel<<<blocks_for(P2), TPB, 0, st>>>(R[cur].p, node[cur].p, src.p, m, P2, R[cur ^ 1].p, node[cur ^ 1].p);
      SK_CUDA(launched(3));
      sq[cur].release();
      cur ^= 1;
      S = m;
      P = P2;
      compactions++;
    }
    const uint64_t nt = P / TILE, n_tiles = nt * (nt + 1) / 2;
    nj_scan_kernel<<<(unsigned)std::min<uint64_t>(n_tiles, scan_cap), SCAN_TPB, 0, st>>>(sq[cur].p, P, R[cur].p, m, n_tiles, part.p, arrived.p, sel.p);
    nj_update_kernel<<<blocks_for(S), TPB, 0, st>>>(sq[cur].p, P, S, R[cur].p, node[cur].p, sel.p, n, t, d_joins.p);
    SK_CUDA(launched(2));
  }
  nj_last_kernel<<<1, 1, 0, st>>>(sq[cur].p, P, S, R[cur].p, node[cur].p, n, d_joins.p);
  SK_CUDA(launched());
  SK_CUDA(cudaMemcpyAsync(joins, d_joins.p, (size_t)(n - 1) * sizeof(sk_nj_join), cudaMemcpyDeviceToHost, st));
  SK_CUDA(cudaStreamSynchronize(st));
  if (stats) { stats->joins = n - 1; stats->compactions = compactions; }
  return SK_OK;
}

}  // namespace

int sk_neighbor_joining(sk_ctx* ctx, uint32_t n_genomes, const sk_ani_result* results, uint64_t n_results, sk_nj_join* joins,
                        sk_nj_stats* stats) {
  if (!ctx) return SK_ERR_PARAM;
  if ((n_results && !results) || (n_genomes > 1 && !joins)) { ctx->err = std::string(WHO) + ": NULL argument"; return SK_ERR_PARAM; }
  SK_CUDA(cudaSetDevice(ctx->device));
  const auto t0 = std::chrono::steady_clock::now();
  const int rc = nj_impl(ctx, n_genomes, results, n_results, joins, stats);
  if (rc == SK_OK && stats) stats->t_device = std::chrono::duration<double>(std::chrono::steady_clock::now() - t0).count();
  return rc;
}
