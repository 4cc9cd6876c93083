"""sk_neighbor_joining on the GPU (skani_b200.neighbor_joining) against tests/nj_ref.py: the join table (a, b and the float64
lengths) bit for bit on random sparse graphs up to 1 500 genomes, tie-heavy graphs (all missing, families with one ANI) and
sizes around the scan tile and the compaction edges; exact recovery of random additive trees up to 4 000 genomes from dense
rows, through many compactions; row order; and every refusal."""
import numpy as np
import pytest

import cluster_ref as CR
import nj_ref as N

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def ctx():
    import skani_b200 as sk
    c = sk.Context(0)
    yield c
    c.close()


def nj(ctx, n, a, b, ani):
    import skani_b200 as sk
    joins, st = sk.neighbor_joining(ctx, n, CR.as_results(a, b, ani))
    assert st.joins == max(n - 1, 0) and joins.dtype == N.NJ_JOIN_DTYPE
    return joins, st


def check(ctx, n, a, b, ani):
    joins, st = nj(ctx, n, a, b, ani)
    want = N.nj_results(n, a, b, ani)
    assert np.array_equal(joins["a"], want["a"]) and np.array_equal(joins["b"], want["b"]), n
    assert np.array_equal(joins["len_a"].view(np.uint64), want["len_a"].view(np.uint64)), n
    assert np.array_equal(joins["len_b"].view(np.uint64), want["len_b"].view(np.uint64)), n
    return st


@pytest.mark.parametrize("n", [2, 3, 4, 31, 32, 33, 63, 64, 65, 127, 128, 129, 300, 700])
def test_sizes_around_tile_and_compaction(ctx, n):
    rng = np.random.default_rng(n)
    st = check(ctx, *CR.erdos_renyi(rng, n, 4 * n))
    assert st.compactions == (0 if n <= 64 else st.compactions) and (n < 100 or st.compactions > 0)


@pytest.mark.parametrize("seed", range(4))
def test_random_sparse(ctx, seed):
    rng = np.random.default_rng(1000 + seed)
    n = [500, 900, 1200, 1500][seed]
    if seed % 2:
        check(ctx, *CR.families(rng, n, int(rng.integers(3, 12)), 2 * n))
    else:
        check(ctx, *CR.erdos_renyi(rng, n, 5 * n))


@pytest.mark.parametrize("n", [2, 3, 5, 64, 65, 200])
def test_all_missing(ctx, n):
    empty = np.zeros(0, np.uint32)
    check(ctx, n, empty, empty, np.zeros(0, np.float32))


@pytest.mark.parametrize("n", [40, 130, 400])
def test_families_with_one_ani(ctx, n):
    rng = np.random.default_rng(n)
    n, a, b, ani = CR.families(rng, n, 5, n // 2)
    check(ctx, n, a, b, np.full(len(a), np.float32(0.97)))


def test_row_order_and_direction_do_not_matter(ctx):
    rng = np.random.default_rng(5)
    n, a, b, ani = CR.families(rng, 300, 6, 300)
    base, _ = nj(ctx, n, a, b, ani)
    o = rng.permutation(len(a))
    again, _ = nj(ctx, n, b[o], a[o], ani[o])
    assert base.tobytes() == again.tobytes()


@pytest.mark.parametrize("n", [50, 500, 1500, 4000])
def test_additive_trees_recovered(ctx, n):
    rng = np.random.default_rng(n)
    D, parent, _ = N.random_additive(rng, n)
    a, b = np.triu_indices(n, 1)
    ani = (1.0 - D[a, b]).astype(np.float32)
    joins, st = nj(ctx, n, a.astype(np.uint32), b.astype(np.uint32), ani)
    parent2, length2 = N.tree_of_joins(n, joins)
    assert N.splits(n, parent2) == N.splits(n, parent)
    assert np.array_equal(N.patristic(n, parent2, length2), D)
    assert st.compactions >= (4 if n >= 1500 else 0)


def test_refusals(ctx):
    import skani_b200 as sk
    from skani_b200.host import SkaniError

    def refused(n, a, b, ani, text):
        with pytest.raises(SkaniError) as e:
            sk.neighbor_joining(ctx, n, CR.as_results(np.array(a, np.uint32), np.array(b, np.uint32), np.array(ani, np.float32)))
        assert "sk_neighbor_joining" in str(e.value) and text in str(e.value), str(e.value)
    refused(3, [0, 1], [1, 3], [0.9, 0.9], "genome id")
    refused(3, [0, 2], [1, 2], [0.9, 0.9], "self pair")
    refused(3, [0, 1], [1, 0], [0.9, 0.95], "listed twice")
    refused(3, [0, 1], [1, 2], [0.9, 1.0001], "ani > 1")
    refused(3, [0, 1], [1, 2], [0.9, np.inf], "ani > 1")
    res = CR.as_results(np.array([0], np.uint32), np.array([1], np.uint32), np.array([0.9], np.float32))
    rc = ctx.L.sk_neighbor_joining(ctx.h, 2, res.ctypes.data, 1, None, None)
    assert rc != 0 and "NULL" in ctx.L.sk_last_error(ctx.h).decode()
    for n in (0, 1):                  # no rows, and joins may be NULL
        assert ctx.L.sk_neighbor_joining(ctx.h, n, None, 0, None, None) == 0
        joins, st = sk.neighbor_joining(ctx, n, CR.as_results([], [], []))
        assert len(joins) == 0 and st.joins == 0
    # ani == 1 is distance 0, and rows that are never edges are ignored
    n, a, b = 4, [0, 1, 2], [1, 2, 3]
    check(ctx, n, np.array(a, np.uint32), np.array(b, np.uint32), np.array([1.0, np.nan, 0.1], np.float32))
