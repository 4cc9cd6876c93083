"""sk_cluster_linkage on the GPU (skani_b200.cluster_linkage) against the round procedure of tests/linkage_ref.py: rep,
cluster, edge, the scipy linkage matrix and the round count bit for bit, for average and complete linkage, in cut and in
dendrogram mode, on Erdos-Renyi graphs, families joined by cross edges, paths (equal ANIs, and ANI decreasing along the
path), stars, equal ANIs and sentinel rows, in three rank orders; row order; a 10^6-row case checked by invariants; every
refusal; and the results of real triangles of synthetic families."""
import ctypes as C

import numpy as np
import pytest

import cluster_ref as CR
import linkage_ref as L
from bench_support import synth

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def ctx():
    import skani_b200 as sk
    c = sk.Context(0)
    yield c
    c.close()


def run(ctx, n, res, rank, method, min_ani, dendrogram):
    import skani_b200 as sk
    return sk.cluster_linkage(ctx, n, res, rank, method=method, min_ani=min_ani, dendrogram=dendrogram)


def check(ctx, n, res, rank, method, min_ani):
    """both modes against the reference; the cut-mode partition equals the dendrogram-mode one"""
    out = {}
    for dendrogram in (False, True):
        rep, cl, edge, Z, st = run(ctx, n, res, rank, method, min_ani, dendrogram)
        erep, ecl, eedge, eZ, erounds = L.rounds(n, res["ref_id"], res["query_id"], res["ani"], rank, method, min_ani, dendrogram)
        assert np.array_equal(rep, erep) and np.array_equal(cl, ecl) and np.array_equal(edge, eedge), (method, dendrogram)
        if dendrogram:
            assert Z.shape == (max(n - 1, 0), 4) and np.array_equal(Z, eZ), method
        else:
            assert Z is None
        assert st.rounds == erounds
        assert st.n_clusters == (int(cl.max()) + 1 if n else 0)
        assert st.n_edges == len(L._edges(None, None, res["ani"]))
        out[dendrogram] = (rep, cl, edge)
    for x, y in zip(out[False], out[True]):
        assert np.array_equal(x, y)
    return out[True]


def decreasing_path(rng, n):
    p = np.stack([np.arange(n - 1), np.arange(1, n)], 1)
    return CR._finish(rng, n, p, np.linspace(0.999, 0.9, n - 1).astype(np.float32))


def graph_of(kind, rng):
    if kind == "erdos_renyi":
        return CR.erdos_renyi(rng, 3000, 12000)
    if kind == "families":
        return CR.families(rng, 2000, 20, 3000, inside=(0.93, 1.0))
    if kind == "path":
        return CR.path(rng, 500)
    if kind == "decreasing_path":
        return decreasing_path(rng, 600)
    if kind == "stars":
        return CR.stars(rng, 1000, 7)
    if kind == "equal":
        n, a, b, ani = CR.families(rng, 600, 12, 800)
        return n, a, b, np.full(len(a), 0.97, np.float32)
    n, a, b, ani = CR.erdos_renyi(rng, 2000, 6000)                  # "special": cut ties, sentinels, isolated genomes
    ani = ani.copy()
    pick = rng.random(len(ani))
    ani[pick < 0.2] = np.float32(0.95)
    ani[(pick >= 0.2) & (pick < 0.25)] = np.float32("nan")
    ani[(pick >= 0.25) & (pick < 0.3)] = np.float32(-1)
    ani[(pick >= 0.3) & (pick < 0.32)] = np.float32(0.1)
    ani[(pick >= 0.32) & (pick < 0.34)] = np.float32(0.3)
    return n + 500, a, b, ani


KINDS = ["erdos_renyi", "families", "path", "decreasing_path", "stars", "equal", "special"]
ORDERS = ["random", "rank", "reverse"]


@pytest.mark.parametrize("kind", KINDS)
@pytest.mark.parametrize("method", L.METHODS)
@pytest.mark.parametrize("order", ORDERS)
def test_families_match_reference(ctx, kind, method, order):
    rng = np.random.default_rng([KINDS.index(kind), L.METHODS.index(method), ORDERS.index(order)])
    n, a, b, ani = graph_of(kind, rng)
    rank = {"random": rng.permutation(n), "rank": np.arange(n), "reverse": np.arange(n)[::-1].copy()}[order]
    res = CR.as_results(a, b, ani)
    for min_ani in (0.95, 0.975):
        check(ctx, n, res, rank, method, min_ani)


def test_result_independent_of_row_order(ctx):
    import skani_b200 as sk
    rng = np.random.default_rng(5)
    n, a, b, ani = CR.families(rng, 4000, 20, 6000)
    rank = rng.permutation(n)
    res = CR.as_results(a, b, ani)
    for method in L.METHODS:
        base = run(ctx, n, res, rank, method, 0.96, True)
        for _ in range(2):
            p = rng.permutation(len(res))
            rep, cl, edge, Z, _ = run(ctx, n, res[p], rank, method, 0.96, True)
            assert np.array_equal(rep, base[0]) and np.array_equal(cl, base[1]) and np.array_equal(Z, base[3])
            moved = edge != sk.host.NO_EDGE
            assert np.array_equal(moved, base[2] != sk.host.NO_EDGE)
            assert np.array_equal(p[edge[moved].astype(np.int64)], base[2][moved].astype(np.int64))


def check_linkage_invariants(Z, n):
    """a valid linkage matrix over n leaves with monotone heights (numpy only)"""
    assert Z.shape == (n - 1, 4)
    a, b, h, size = Z[:, 0].astype(np.int64), Z[:, 1].astype(np.int64), Z[:, 2], Z[:, 3].astype(np.int64)
    j = np.arange(n - 1)
    assert (a < b).all() and (b < n + j).all() and (a >= 0).all()
    used = np.concatenate([a, b])
    assert len(np.unique(used)) == len(used) == 2 * (n - 1)
    sz = np.concatenate([np.ones(n, np.int64), size])
    assert np.array_equal(size, sz[a] + sz[b])
    assert (np.diff(h) >= 0).all() and (h >= 0).all() and h[-1] <= 1.0


def test_large_families_invariants(ctx):
    """100,000 genomes in families of 20 plus cross edges, 1.05 x 10^6 rows: the dendrogram is a valid, monotone linkage
    and its fcluster at 1 - min_ani is the flat partition"""
    from scipy.cluster.hierarchy import fcluster
    rng = np.random.default_rng(17)
    n, a, b, ani = CR.families(rng, 100_000, 20, 100_000, inside=(0.9, 1.0))
    res = CR.as_results(a, b, ani)
    assert len(res) >= 1_000_000
    rank = rng.permutation(n)
    for method in L.METHODS:
        rep, cl, edge, Z, st = run(ctx, n, res, rank, method, 0.96, True)
        check_linkage_invariants(Z, n)
        assert L.partition(fcluster(Z, 1.0 - float(np.float32(0.96)), "distance")) == L.partition(cl)
        rep2, cl2, edge2, _, st2 = run(ctx, n, res, rank, method, 0.96, False)
        assert np.array_equal(rep, rep2) and np.array_equal(cl, cl2) and np.array_equal(edge, edge2)
        assert (rank[rep] <= rank).all() and st.n_clusters == st2.n_clusters == int(cl.max()) + 1
        print("%s linkage of %d genomes, %d rows: %d clusters, %d rounds, %.3f s (cut mode %.3f s)" % (
            method, n, len(res), st.n_clusters, st.rounds, st.t_device, st2.t_device))


def test_star_one_leaf_per_round(ctx):
    """A star merges one leaf per round in average linkage: 3,000 leaves, 3,000 rounds."""
    rng = np.random.default_rng(9)
    n, a, b, ani = CR.stars(rng, 3001, 1)
    ani = L.tie_free(rng, ani, 0.96, 1.0)
    res = CR.as_results(a, b, ani)
    check(ctx, n, res, rng.permutation(n), "average", 0.9)
    _, _, _, _, st = run(ctx, n, res, np.arange(n), "average", 0.9, True)
    assert st.rounds == n - 1


def test_empty_and_edgeless(ctx):
    import skani_b200 as sk
    res0 = np.zeros(0, sk.host.RESULT_DTYPE)
    for method in L.METHODS:
        rep, cl, edge, Z, st = run(ctx, 0, res0, np.zeros(0, np.uint32), method, 0.95, True)
        assert len(rep) == len(cl) == len(edge) == 0 and Z.shape == (0, 4) and st.n_clusters == 0
        rep, cl, edge, Z, st = run(ctx, 1, res0, np.zeros(1, np.uint32), method, 0.95, True)
        assert rep.tolist() == [0] and cl.tolist() == [0] and Z.shape == (0, 4)
        rank = np.array([2, 0, 1, 3], np.uint32)
        for res in (res0, CR.as_results([0, 1, 2], [1, 2, 3], np.array([0.1, np.nan, -1], np.float32))):
            rep, cl, edge, Z, st = run(ctx, 4, res, rank, method, 0.95, True)
            assert np.array_equal(rep, np.arange(4)) and np.array_equal(cl, rank) and (edge == sk.host.NO_EDGE).all()
            assert st.n_clusters == 4 and st.n_edges == 0 and st.rounds == 0
            # leftovers joined at 1.0 in rank order: genomes 1, 2, 0, 3
            assert Z.tolist() == [[1, 2, 1.0, 2], [0, 4, 1.0, 3], [3, 5, 1.0, 4]]


def test_refusals(ctx):
    import skani_b200 as sk
    from skani_b200 import _lib
    ok = CR.as_results([0, 1], [1, 2], np.array([0.99, 0.98], np.float32))
    rank = np.arange(3, dtype=np.uint32)
    cases = [
        (CR.as_results([0, 3], [1, 1], np.array([0.99, 0.5], np.float32)), rank, 0.95, "n_genomes"),
        (CR.as_results([0, 2], [1, 2], np.array([0.99, 0.99], np.float32)), rank, 0.95, "self pair"),
        (CR.as_results([0, 1], [1, 0], np.array([0.99, 0.5], np.float32)), rank, 0.95, "listed twice"),
        (ok, np.array([0, 0, 1], np.uint32), 0.95, "permutation"),
        (CR.as_results([0, 1], [1, 2], np.array([0.99, 2.0], np.float32)), rank, 0.95, "ani >= 2"),
        (CR.as_results([0, 1], [1, 2], np.array([np.inf, 0.9], np.float32)), rank, 0.95, "ani >= 2"),
        (ok, rank, 0.1, "min_ani"),
        (ok, rank, 1.01, "min_ani"),
        (ok, rank, float("nan"), "min_ani"),
    ]
    for res, rk, min_ani, msg in cases:
        for method in L.METHODS:
            with pytest.raises(sk.host.SkaniError, match=msg):
                run(ctx, 3, res, rk, method, min_ani, False)
    with pytest.raises(ValueError):
        run(ctx, 3, ok, rank, "single", 0.95, False)
    # through the C ABI: an unknown method, NULL outputs, NULL merges in dendrogram mode
    st = _lib.ClusterStats()
    out32 = np.zeros(3, np.uint32); out64 = np.zeros(3, np.uint64)
    merges = np.zeros(2, sk.host.MERGE_DTYPE)

    def call(lp, i=None, dendro_merges=True):
        args = [ctx.h, 3, ok.ctypes.data, len(ok), rank.ctypes.data, C.byref(lp), out32.ctypes.data, out32.ctypes.data, out64.ctypes.data,
                merges.ctypes.data if dendro_merges else None, C.byref(st)]
        if i is not None:
            args[i] = None
        return ctx.L.sk_cluster_linkage(*args)
    assert call(_lib.LinkageParams(0.95, 2, 0)) == -2 and "method" in ctx.L.sk_last_error(ctx.h).decode()
    assert call(_lib.LinkageParams(0.95, 0, 1), dendro_merges=False) == -2 and "NULL" in ctx.L.sk_last_error(ctx.h).decode()
    assert call(_lib.LinkageParams(0.95, 0, 0), dendro_merges=False) == 0          # merges may be NULL in cut mode
    for i in (5, 6, 7, 8):
        assert call(_lib.LinkageParams(0.95, 0, 1), i) == -2 and "NULL" in ctx.L.sk_last_error(ctx.h).decode()
    assert call(_lib.LinkageParams(0.95, 1, 1), 10) == 0                            # stats may be NULL
    # the context still works after every refusal
    check(ctx, 3, ok, rank, "average", 0.95)


def test_real_triangle_results(ctx):
    """Triangles of synthetic families (bench_support.synth), clustered at cuts between the printed ANIs."""
    import skani_b200 as sk
    n, L_, G = 40, 200_000, 5
    bases, off, goc = synth.generate(0, n, L_, G=G)
    units, nmask, lens = sk.pack_contigs(ctx.L, bases, off)
    res, _ = sk.triangle_2bit(ctx, units, nmask, lens, goc, n)
    res = res[res["ani"] > np.float32(0.1)]
    assert len(res) > n
    total = np.bincount(goc, weights=lens.astype(np.float64), minlength=n)
    order = np.lexsort((np.arange(n), -total))
    rank = np.empty(n, np.uint32); rank[order] = np.arange(n)
    printed = np.unique(np.round(res["ani"].astype(np.float64) * 100, 2))
    mids = (printed[:-1] + printed[1:]) / 2
    for t in [mids[len(mids) // 4], mids[len(mids) // 2], mids[3 * len(mids) // 4], 95.0]:
        for method in L.METHODS:
            check(ctx, n, res, rank, method, float(np.float32(t / 100)))
