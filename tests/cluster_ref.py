"""Python references of sk_cluster (include/skani_b200.h) and the graph families its tests and tools/bench_cluster.py use.

greedy: a sequential loop in rank order; single linkage: scipy.sparse.csgraph.connected_components with the smallest-rank
member as representative.  Both take (n, a, b, ani, min_ani, rank) where row i joins a[i] and b[i]; they return
(rep, cluster, edge) as sk_cluster defines them (edge = row index, NO_EDGE when there is none)."""
import numpy as np

NO_EDGE = np.uint64(0xFFFFFFFFFFFFFFFF)


def edge_rows(ani, min_ani):
    ani = np.asarray(ani, np.float32)
    with np.errstate(invalid="ignore"):
        return np.nonzero((ani > np.float32(0.1)) & (ani >= np.float32(min_ani)))[0]


def _csr(n, a, b, rows):
    src = np.concatenate([a[rows], b[rows]]).astype(np.int64)
    dst = np.concatenate([b[rows], a[rows]]).astype(np.int64)
    row = np.concatenate([rows, rows]).astype(np.int64)
    o = np.lexsort((dst, src))
    src, dst, row = src[o], dst[o], row[o]
    off = np.searchsorted(src, np.arange(n + 1))
    return off, src, dst, row


def _number(n, rank, rep, is_rep):
    order = np.argsort(rank, kind="stable")
    cid = np.cumsum(is_rep[order]) - 1             # cluster id by rank position
    return cid[np.asarray(rank, np.int64)[rep]].astype(np.uint32)


def greedy(n, a, b, ani, min_ani, rank):
    a = np.asarray(a, np.int64); b = np.asarray(b, np.int64); ani = np.asarray(ani, np.float32)
    rank = np.asarray(rank, np.int64)
    rows = edge_rows(ani, min_ani)
    off, src, dst, row = _csr(n, a, b, rows)
    is_rep = np.zeros(n, bool)
    for v in np.argsort(rank, kind="stable"):
        if not is_rep[dst[off[v]:off[v + 1]]].any():
            is_rep[v] = True
    rep = np.arange(n, dtype=np.int64)
    edge = np.full(n, NO_EDGE, np.uint64)
    cand = np.nonzero(~is_rep[src] & is_rep[dst])[0]          # member -> representative neighbour
    if len(cand):
        s, d, r = src[cand], dst[cand], row[cand]
        o = np.lexsort((rank[d], -ani[r].astype(np.float64), s))   # per member: highest ANI, then smallest rank
        s, d, r = s[o], d[o], r[o]
        first = np.ones(len(s), bool)
        first[1:] = s[1:] != s[:-1]
        rep[s[first]] = d[first]
        edge[s[first]] = r[first].astype(np.uint64)
    return rep.astype(np.uint32), _number(n, rank, rep, is_rep), edge


def single_linkage(n, a, b, ani, min_ani, rank):
    import scipy.sparse as sp
    from scipy.sparse.csgraph import connected_components
    a = np.asarray(a, np.int64); b = np.asarray(b, np.int64)
    rank = np.asarray(rank, np.int64)
    rows = edge_rows(ani, min_ani)
    g = sp.coo_matrix((np.ones(len(rows), np.int8), (a[rows], b[rows])), shape=(n, n)).tocsr()
    _, label = connected_components(g, directed=False)
    best = np.full(label.max() + 1 if n else 0, np.iinfo(np.int64).max, np.int64)
    np.minimum.at(best, label, rank)
    order = np.argsort(rank, kind="stable")
    rep = order[best[label]]
    is_rep = rep == np.arange(n)
    edge = np.full(n, NO_EDGE, np.uint64)
    key = np.minimum(a[rows], b[rows]) * (1 << 32) + np.maximum(a[rows], b[rows])
    o = np.argsort(key)
    key, krow = key[o], rows[o]
    mem = np.nonzero(~is_rep)[0]
    want = np.minimum(mem, rep[mem]) * (1 << 32) + np.maximum(mem, rep[mem])
    at = np.searchsorted(key, want)
    hit = (at < len(key)) & (key[np.minimum(at, max(len(key) - 1, 0))] == want) if len(key) else np.zeros(len(mem), bool)
    edge[mem[hit]] = krow[at[hit]].astype(np.uint64)
    return rep.astype(np.uint32), _number(n, rank, rep, is_rep), edge


def reference(n, a, b, ani, min_ani, rank, single=False):
    return (single_linkage if single else greedy)(n, a, b, ani, min_ani, rank)


# ---- graph families: (n, a, b, ani) with unique unordered pairs, rows in random order and direction
def _finish(rng, n, pairs, ani):
    pairs = np.asarray(pairs, np.int64).reshape(-1, 2)
    lo, hi = pairs.min(axis=1), pairs.max(axis=1)
    keep = lo != hi
    key, idx = np.unique(lo[keep] * (1 << 32) + hi[keep], return_index=True)
    ani = np.asarray(ani, np.float32)[keep][idx]
    a, b = (key >> 32).astype(np.uint32), (key & 0xFFFFFFFF).astype(np.uint32)
    flip = rng.random(len(a)) < 0.5
    a, b = np.where(flip, b, a), np.where(flip, a, b)
    o = rng.permutation(len(a))
    return n, a[o], b[o], ani[o]


def rand_ani(rng, m, lo=0.90, hi=1.0):
    return (lo + (hi - lo) * rng.random(m)).astype(np.float32)


def erdos_renyi(rng, n, m):
    p = rng.integers(0, n, size=(m, 2))
    return _finish(rng, n, p, rand_ani(rng, m))


def families(rng, n, size, cross, inside=(0.96, 1.0)):
    """cliques of `size` consecutive genomes (ANI in `inside`) plus `cross` random pairs (ANI 0.90-1.0)"""
    f = np.arange(n) // size
    starts = np.arange(0, n, size)
    pa, pb = [], []
    for i in range(size):
        for j in range(i + 1, size):
            x = starts + i; y = starts + j
            ok = y < n
            pa.append(x[ok]); pb.append(y[ok])
    pa = np.concatenate(pa) if pa else np.zeros(0, np.int64)
    pb = np.concatenate(pb) if pb else np.zeros(0, np.int64)
    c = rng.integers(0, n, size=(cross, 2))
    c = c[f[c[:, 0]] != f[c[:, 1]]]
    pairs = np.concatenate([np.stack([pa, pb], 1), c])
    ani = np.concatenate([rand_ani(rng, len(pa), *inside), rand_ani(rng, len(c))])
    return _finish(rng, n, pairs, ani)


def path(rng, n, ani=0.99):
    p = np.stack([np.arange(n - 1), np.arange(1, n)], 1)
    return _finish(rng, n, p, np.full(n - 1, ani, np.float32))


def stars(rng, n, centres):
    v = np.arange(centres, n)
    return _finish(rng, n, np.stack([v % centres, v], 1), rand_ani(rng, len(v)))


def as_results(a, b, ani):
    """a RESULT_DTYPE array whose rows carry (ref_id, query_id, ani); af_ref = 0.5, af_query = 0.25"""
    from skani_b200.host import RESULT_DTYPE
    r = np.zeros(len(a), RESULT_DTYPE)
    r["ref_id"], r["query_id"], r["ani"] = a, b, ani
    r["af_ref"] = np.float32(0.5); r["af_query"] = np.float32(0.25)
    return r
