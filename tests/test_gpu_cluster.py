"""sk_cluster on the GPU (skani_b200.cluster) against the Python references of tests/cluster_ref.py: greedy representatives
(a sequential loop) and single linkage (scipy connected components), on Erdos-Renyi graphs, families joined by cross edges,
paths, stars, equal ANIs, ani == min_ani and sentinel rows, up to 200,000 genomes and 5 x 10^6 edges; every refusal; and the
results of real triangles of synthetic families."""
import time

import numpy as np
import pytest

import cluster_ref as R
from bench_support import synth

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def ctx():
    import skani_b200 as sk
    c = sk.Context(0)
    yield c
    c.close()


def check(ctx, n, a, b, ani, rank, min_ani, single, res=None):
    import skani_b200 as sk
    res = R.as_results(a, b, ani) if res is None else res
    rep, cl, edge, st = sk.cluster(ctx, n, res, rank, min_ani=min_ani, single_linkage=single)
    erep, ecl, eedge = R.reference(n, res["ref_id"], res["query_id"], res["ani"], min_ani, rank, single)
    bad = np.nonzero((rep != erep) | (cl != ecl) | (edge != eedge))[0]
    assert len(bad) == 0, ("first differing genome", int(bad[0]), int(rep[bad[0]]), int(erep[bad[0]]), int(cl[bad[0]]), int(ecl[bad[0]]),
                           int(edge[bad[0]]), int(eedge[bad[0]]))
    assert st.n_clusters == (int(cl.max()) + 1 if n else 0) == int((rep == np.arange(n)).sum())
    assert st.n_edges == len(R.edge_rows(res["ani"], min_ani))
    has = edge != sk.host.NO_EDGE
    rows = res[edge[has].astype(np.int64)]
    g = np.nonzero(has)[0]
    assert np.array_equal(np.minimum(rows["ref_id"], rows["query_id"]), np.minimum(g, rep[has]))
    assert np.array_equal(np.maximum(rows["ref_id"], rows["query_id"]), np.maximum(g, rep[has]))
    return rep, cl, edge, st


def families_of(kind, rng):
    if kind == "erdos_renyi":
        return R.erdos_renyi(rng, 3000, 12000)
    if kind == "families":
        return R.families(rng, 2000, 20, 3000, inside=(0.93, 1.0))
    if kind == "path":
        return R.path(rng, 500)
    if kind == "stars":
        return R.stars(rng, 1000, 7)
    if kind == "equal":
        n, a, b, ani = R.families(rng, 600, 12, 800)
        return n, a, b, np.full(len(a), 0.97, np.float32)
    n, a, b, ani = R.erdos_renyi(rng, 2000, 6000)                  # "special": threshold ties, sentinels, isolated genomes
    ani = ani.copy()
    pick = rng.random(len(ani))
    ani[pick < 0.2] = np.float32(0.95)
    ani[(pick >= 0.2) & (pick < 0.25)] = np.float32("nan")
    ani[(pick >= 0.25) & (pick < 0.3)] = np.float32(-1)
    ani[(pick >= 0.3) & (pick < 0.32)] = np.float32(0.1)
    return n + 500, a, b, ani


KINDS = ["erdos_renyi", "families", "path", "stars", "equal", "special"]
ORDERS = ["random", "rank", "reverse"]


@pytest.mark.parametrize("kind", KINDS)
@pytest.mark.parametrize("single", [False, True])
@pytest.mark.parametrize("order", ORDERS)
def test_families_match_reference(ctx, kind, single, order):
    rng = np.random.default_rng([KINDS.index(kind), int(single), ORDERS.index(order)])
    n, a, b, ani = families_of(kind, rng)
    rank = {"random": rng.permutation(n), "rank": np.arange(n), "reverse": np.arange(n)[::-1].copy()}[order]
    for min_ani in (0.95, 0.975):
        check(ctx, n, a, b, ani, rank, min_ani, single)


def test_result_independent_of_row_order(ctx):
    import skani_b200 as sk
    rng = np.random.default_rng(5)
    n, a, b, ani = R.families(rng, 4000, 20, 6000)
    rank = rng.permutation(n)
    res = R.as_results(a, b, ani)
    base = sk.cluster(ctx, n, res, rank)
    for _ in range(3):
        p = rng.permutation(len(res))
        rep, cl, edge, _ = sk.cluster(ctx, n, res[p], rank)
        assert np.array_equal(rep, base[0]) and np.array_equal(cl, base[1])
        moved = edge != sk.host.NO_EDGE
        assert np.array_equal(np.nonzero(moved)[0], np.nonzero(base[2] != sk.host.NO_EDGE)[0])
        assert np.array_equal(p[edge[moved].astype(np.int64)], base[2][moved].astype(np.int64))


@pytest.mark.parametrize("single", [False, True])
def test_large_families_and_cross_edges(ctx, single):
    """200,000 genomes: families of 20 (1.9 M edges inside) and 3.1 M random cross edges, 5 M rows in all."""
    rng = np.random.default_rng(11)
    n, a, b, ani = R.families(rng, 200_000, 20, 3_100_000, inside=(0.95, 1.0))
    assert len(a) > 4_900_000
    check(ctx, n, a, b, ani, rng.permutation(n), 0.97, single)


def test_path_in_rank_order(ctx):
    """The greedy worst case: a 100,000-genome path ranked along the path decides about one genome per round."""
    rng = np.random.default_rng(3)
    n, a, b, ani = R.path(rng, 100_000)
    t = time.perf_counter()
    _, cl, _, st = check(ctx, n, a, b, ani, np.arange(n), 0.95, False)
    print("path of %d genomes in rank order: %d rounds, %.3f s in sk_cluster (%.3f s with the reference)" % (n, st.rounds, st.t_device,
                                                                                                         time.perf_counter() - t))
    assert st.n_clusters == n // 2 and st.rounds >= 1
    check(ctx, n, a, b, ani, np.arange(n), 0.95, True)


def test_empty_and_edgeless(ctx):
    import skani_b200 as sk
    res0 = np.zeros(0, sk.host.RESULT_DTYPE)
    rep, cl, edge, st = sk.cluster(ctx, 0, res0, np.zeros(0, np.uint32))
    assert len(rep) == len(cl) == len(edge) == 0 and st.n_clusters == 0 and st.n_edges == 0
    rank = np.array([2, 0, 1, 3], np.uint32)
    for res in (res0, R.as_results([0, 1, 2], [1, 2, 3], np.array([0.5, np.nan, -1], np.float32))):
        for single in (False, True):
            rep, cl, edge, st = sk.cluster(ctx, 4, res, rank, single_linkage=single)
            assert np.array_equal(rep, np.arange(4)) and np.array_equal(cl, rank) and (edge == sk.host.NO_EDGE).all()
            assert st.n_clusters == 4 and st.n_edges == 0


def test_refusals(ctx):
    import ctypes as C
    import skani_b200 as sk
    from skani_b200 import _lib
    ok = R.as_results([0, 1], [1, 2], np.array([0.99, 0.98], np.float32))
    rank = np.arange(3, dtype=np.uint32)
    cases = [
        (R.as_results([0, 3], [1, 1], np.array([0.99, 0.5], np.float32)), rank, "n_genomes"),     # id >= n (not even an edge)
        (R.as_results([0, 2], [1, 2], np.array([0.99, 0.99], np.float32)), rank, "self pair"),
        (R.as_results([0, 1], [1, 0], np.array([0.99, 0.98], np.float32)), rank, "listed twice"),
        (ok, np.array([0, 0, 1], np.uint32), "permutation"),
        (ok, np.array([0, 1, 3], np.uint32), "permutation"),
    ]
    for res, rk, msg in cases:
        with pytest.raises(sk.host.SkaniError, match=msg):
            sk.cluster(ctx, 3, res, rk)
        with pytest.raises(sk.host.SkaniError, match=msg):
            sk.cluster(ctx, 3, res, rk, single_linkage=True)
    # NULL outputs and parameters through the C ABI
    cp, st = _lib.ClusterParams(0.95, 0), _lib.ClusterStats()
    out32 = np.zeros(3, np.uint32); out64 = np.zeros(3, np.uint64)
    args = [ctx.h, 3, ok.ctypes.data, len(ok), rank.ctypes.data, C.byref(cp), out32.ctypes.data, out32.ctypes.data, out64.ctypes.data, C.byref(st)]
    for i in (5, 6, 7, 8):
        bad = list(args)
        bad[i] = None
        assert ctx.L.sk_cluster(*bad) == -2
        assert "NULL" in ctx.L.sk_last_error(ctx.h).decode()
    assert ctx.L.sk_cluster(*args[:9], None) == 0      # stats may be NULL
    # the context still works after every refusal
    check(ctx, 3, ok["ref_id"], ok["query_id"], ok["ani"], rank, 0.95, False)


def test_real_triangle_results(ctx):
    """Triangles of synthetic families (bench_support.synth) clustered at thresholds between the printed ANIs."""
    import skani_b200 as sk
    n, L, G = 40, 200_000, 5
    bases, off, goc = synth.generate(0, n, L, G=G)
    units, nmask, lens = sk.pack_contigs(ctx.L, bases, off)
    res, _ = sk.triangle_2bit(ctx, units, nmask, lens, goc, n)
    res = res[res["ani"] > np.float32(0.1)]
    assert len(res) > n
    total = np.bincount(goc, weights=lens.astype(np.float64), minlength=n)
    order = np.lexsort((np.arange(n), -total))                  # longest first, ties by genome index
    rank = np.empty(n, np.uint32); rank[order] = np.arange(n)
    printed = np.unique(np.round(res["ani"].astype(np.float64) * 100, 2))
    mids = (printed[:-1] + printed[1:]) / 2
    for t in [mids[len(mids) // 4], mids[len(mids) // 2], mids[3 * len(mids) // 4], 95.0]:
        for single in (False, True):
            check(ctx, n, None, None, None, rank, np.float32(t / 100), single, res=res)
