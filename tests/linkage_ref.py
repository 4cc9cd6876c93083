"""Python references of sk_cluster_linkage (include/skani_b200.h) with exact Python-int arithmetic.

rounds(): the round procedure the header defines (reciprocal best partners, ties to the smaller id, deactivation), returning
(rep, cluster, edge, Z, rounds) exactly as the library does.  sequential_hac(): naive sequential agglomeration (always the
globally best qualifying pair, values as Fractions) for small n, the yardstick for inputs without ties.  Rows: row i joins
a[i] and b[i] with ani[i]; the edges are the rows with ani > 0.1, min_ani is the cut only."""
import math
from fractions import Fraction

import numpy as np

import cluster_ref as CR

NO_EDGE = CR.NO_EDGE
METHODS = ("average", "complete")


def q_of(ani):
    """ani * 2^27 as an exact int (every float32 in (0.1, 2) is a multiple of 2^-27)"""
    x = float(np.float32(ani)) * 2.0 ** 27
    assert x == int(x)
    return int(x)


def _edges(a, b, ani):
    ani = np.asarray(ani, np.float32)
    with np.errstate(invalid="ignore"):
        rows = np.nonzero(ani > np.float32(0.1))[0]
    return rows


def _value(method, v, na, nb):
    s, cnt, minq = v
    if method == "average":
        return s, na * nb
    return (minq if cnt == na * nb else 0), 1


def _better(x, y):
    """(s, p, id) x beats y: larger value, then smaller id"""
    l, r = x[0] * y[1], y[0] * x[1]
    return l > r or (l == r and x[2] < y[2])


def _qualifies(s, p, qcut, dendrogram):
    return s > 0 if dendrogram else s >= qcut * p


def _flat(n, a, b, rows, rank, parent):
    """rep / cluster / edge from parent[] in rank space (parent[r] <= r)"""
    def find(r):
        while parent[r] != r:
            r = parent[r]
        return r
    rank = np.asarray(rank, np.int64)
    order = np.empty(n, np.int64); order[rank] = np.arange(n)
    rep = np.array([order[find(int(rank[g]))] for g in range(n)], np.int64)
    is_rep = rep == np.arange(n)
    where = {}
    for i in rows:
        where[(min(int(a[i]), int(b[i])), max(int(a[i]), int(b[i])))] = int(i)
    edge = np.full(n, NO_EDGE, np.uint64)
    for g in range(n):
        if rep[g] != g:
            i = where.get((min(g, int(rep[g])), max(g, int(rep[g]))))
            if i is not None:
                edge[g] = np.uint64(i)
    return rep.astype(np.uint32), CR._number(n, rank, rep, is_rep), edge


def linkage_matrix(n, rank, merges):
    """scipy Z from merges (s, p, round, A, B, size) in rank space: sorted by (value desc, round, A), leftovers joined at
    1.0 in id order"""
    rank = np.asarray(rank, np.int64)
    node = [0] * n
    for g in range(n):
        node[int(rank[g])] = g
    members = [1] * n
    gone = [False] * n
    Z = []

    def join(x, y, h, size):
        Z.append((min(node[x], node[y]), max(node[x], node[y]), h, size))
        node[x] = n + len(Z) - 1
        members[x] = size
        gone[y] = True
    for s, p, rd, A, B, size in sorted(merges, key=lambda m: (-Fraction(m[0], m[1]), m[2], m[3])):
        join(A, B, 1.0 - float(s) / math.ldexp(float(p), 27), size)
    first = None
    for r in range(n):
        if gone[r]:
            continue
        if first is None:
            first = r
        else:
            join(first, r, 1.0, members[first] + members[r])
    return np.array(Z, np.float64).reshape(-1, 4)


def rounds(n, a, b, ani, rank, method="average", min_ani=0.95, dendrogram=False):
    """the library's round procedure; returns (rep, cluster, edge, Z or None, rounds that merged)"""
    a = np.asarray(a, np.int64); b = np.asarray(b, np.int64)
    rank = np.asarray(rank, np.int64)
    rows = _edges(a, b, ani)
    qcut = q_of(min_ani)
    nb = {}                                      # nb[A][B] = [s, cnt, minq], both directions, rank space
    for i in rows:
        x, y, q = int(rank[a[i]]), int(rank[b[i]]), q_of(ani[i])
        nb.setdefault(x, {})[y] = (q, 1, q)
        nb.setdefault(y, {})[x] = (q, 1, q)
    size = [1] * n
    parent = list(range(n))
    merges = []
    rd = last = 0
    while nb:
        best = {}
        for A, part in nb.items():
            cand = None
            for B, v in part.items():
                s, p = _value(method, v, size[A], size[B])
                if cand is None or _better((s, p, B), cand):
                    cand = (s, p, B)
            best[A] = cand[2] if _qualifies(cand[0], cand[1], qcut, dendrogram) else None
        lab = {}
        for A, B in best.items():
            if B is None:
                lab[A] = None
            elif best[B] == A:
                lab[A] = min(A, B)
            else:
                lab[A] = A
        new_size = list(size)
        for A, B in best.items():
            if B is not None and best[B] == A and A < B:
                s, p = _value(method, nb[A][B], size[A], size[B])
                merges.append((s, p, rd, A, B, size[A] + size[B]))
                if _qualifies(s, p, qcut, False):
                    parent[B] = A
                new_size[A] = size[A] + size[B]
                last = rd + 1
        size = new_size
        nxt = {}
        for A, part in nb.items():
            for B, v in part.items():
                x, y = lab[A], lab[B]
                if x is None or y is None or x == y:
                    continue
                d = nxt.setdefault(x, {})
                if y in d:
                    w = d[y]
                    d[y] = (w[0] + v[0], w[1] + v[1], min(w[2], v[2]))
                else:
                    d[y] = v
        nb = nxt
        rd += 1
        assert rd <= n + 1
    rep, cl, edge = _flat(n, a, b, rows, rank, parent)
    Z = linkage_matrix(n, rank, merges) if dendrogram else None
    return rep, cl, edge, Z, last


def sequential_hac(n, a, b, ani, rank, method="average", min_ani=0.95, dendrogram=False):
    """naive exact sequential HAC: always merge the globally most similar pair (Fractions), while it qualifies.  Returns
    (rep, cluster, edge, Z or None); for inputs without ties it equals rounds()."""
    a = np.asarray(a, np.int64); b = np.asarray(b, np.int64)
    rank = np.asarray(rank, np.int64)
    rows = _edges(a, b, ani)
    qcut = Fraction(q_of(min_ani))
    sim = {}
    for i in rows:
        x, y = int(rank[a[i]]), int(rank[b[i]])
        sim[(x, y)] = sim[(y, x)] = q_of(ani[i])
    clusters = {r: [r] for r in range(n)}
    parent = list(range(n))
    merges = []

    def value(A, B):
        qs = [sim.get((x, y)) for x in clusters[A] for y in clusters[B]]
        if method == "average":
            return Fraction(sum(q for q in qs if q is not None), len(qs))
        return Fraction(0) if any(q is None for q in qs) else Fraction(min(qs))
    step = 0
    while len(clusters) > 1:
        ids = sorted(clusters)
        top = None
        for i, A in enumerate(ids):
            for B in ids[i + 1:]:
                v = value(A, B)
                if top is None or v > top[0]:
                    top = (v, A, B)
        v, A, B = top
        if not (v > 0 if dendrogram else v >= qcut):
            break
        merges.append((v.numerator, v.denominator, step, A, B, len(clusters[A]) + len(clusters[B])))
        if v >= qcut:
            parent[B] = A
        clusters[A] += clusters.pop(B)
        step += 1
    rep, cl, edge = _flat(n, a, b, rows, rank, parent)
    Z = linkage_matrix(n, rank, merges) if dendrogram else None
    return rep, cl, edge, Z


def tie_free(rng, ani, lo=0.90, hi=1.0):
    """the same order of ANIs, made pairwise distinct (spacing far above a float32 ulp)"""
    m = len(ani)
    vals = lo + (hi - lo) * (np.arange(m) + 0.5) / max(m, 1)
    out = np.empty(m, np.float32)
    out[np.argsort(np.asarray(ani, np.float64) + 1e-12 * rng.random(m), kind="stable")] = vals.astype(np.float32)
    return out


def dense_similarity(n, a, b, ani):
    """n x n float64 similarity (1 on the diagonal, 0 for pairs without an edge) for scipy"""
    S = np.zeros((n, n))
    rows = _edges(a, b, ani)
    S[np.asarray(a)[rows], np.asarray(b)[rows]] = np.asarray(ani, np.float32)[rows].astype(np.float64)
    S[np.asarray(b)[rows], np.asarray(a)[rows]] = np.asarray(ani, np.float32)[rows].astype(np.float64)
    np.fill_diagonal(S, 1.0)
    return S


def partition(labels):
    """a partition as a set of frozensets of indices"""
    groups = {}
    for i, x in enumerate(np.asarray(labels).tolist()):
        groups.setdefault(x, []).append(i)
    return {frozenset(g) for g in groups.values()}
