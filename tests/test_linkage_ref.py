"""The Python reference of sk_cluster_linkage (tests/linkage_ref.py) on the CPU: its round procedure equals naive sequential
HAC on 240 random graphs without ties (n <= 60, several families), and its dendrogram equals scipy's average / complete
linkage of the dense 1 - similarity matrix (cophenetic distances to 1e-12, flat clusters at cuts away from merge heights)
up to 2,000 genomes."""
import numpy as np
import pytest

import cluster_ref as CR
import linkage_ref as L

FAMILIES = ["erdos_renyi", "families", "path", "stars", "dense"]


def graph(kind, rng, n):
    if kind == "erdos_renyi":
        g = CR.erdos_renyi(rng, n, 2 * n)
    elif kind == "families":
        g = CR.families(rng, n, int(rng.integers(2, 9)), n)
    elif kind == "path":
        g = CR.path(rng, n)
    elif kind == "stars":
        g = CR.stars(rng, n, int(rng.integers(1, 4)))
    else:
        g = CR.erdos_renyi(rng, n, n * n // 3)
    n, a, b, ani = g
    return n, a, b, L.tie_free(rng, ani, 0.85 + 0.1 * rng.random(), 1.0)


@pytest.mark.parametrize("method", L.METHODS)
def test_rounds_equal_sequential_hac(method):
    from scipy.cluster.hierarchy import cophenet
    rng = np.random.default_rng(L.METHODS.index(method))
    cases = 0
    for i in range(120):
        kind = FAMILIES[i % len(FAMILIES)]
        n = int(rng.integers(2, 61))
        n, a, b, ani = graph(kind, rng, n)
        rank = rng.permutation(n)
        min_ani = float(np.float32(0.9 + 0.08 * rng.random()))
        for dendrogram in (False, True):
            got = L.rounds(n, a, b, ani, rank, method, min_ani, dendrogram)
            exp = L.sequential_hac(n, a, b, ani, rank, method, min_ani, dendrogram)
            for x, y in zip(got[:3], exp[:3]):
                assert np.array_equal(x, y), (kind, n, method, dendrogram)
            if dendrogram:      # merges of equal value may be listed in either order: then the cophenetic distances decide
                Zg, Ze = got[3], exp[3]
                if len(np.unique(Ze[:, 2][Ze[:, 2] < 1.0])) == int((Ze[:, 2] < 1.0).sum()):
                    assert np.array_equal(Zg, Ze), (kind, n, method)
                else:
                    assert np.array_equal(cophenet(Zg), cophenet(Ze)), (kind, n, method)
        cases += 1
    assert cases == 120


def check_scipy(n, a, b, ani, method, cuts):
    from scipy.cluster.hierarchy import cophenet, fcluster, is_valid_linkage, linkage
    from scipy.spatial.distance import squareform
    rank = np.arange(n)
    _, cl, _, Z, _ = L.rounds(n, a, b, ani, rank, method, 0.95, True)
    assert is_valid_linkage(Z)
    D = 1.0 - L.dense_similarity(n, a, b, ani)
    np.fill_diagonal(D, 0.0)
    Zs = linkage(squareform(D, checks=False), method)
    assert np.max(np.abs(cophenet(Z) - cophenet(Zs))) <= 1e-12
    heights = np.unique(Z[:, 2])
    checked = 0
    for t in cuts:
        if len(heights) and np.min(np.abs(heights - (1.0 - t))) < 1e-9:
            continue
        _, cl, _, _, _ = L.rounds(n, a, b, ani, rank, method, float(np.float32(t)), False)
        exp = fcluster(Zs, 1.0 - float(np.float32(t)), "distance")
        assert L.partition(cl) == L.partition(exp), (method, t)
        assert L.partition(fcluster(Z, 1.0 - float(np.float32(t)), "distance")) == L.partition(cl)
        checked += 1
    assert checked


@pytest.mark.parametrize("method", L.METHODS)
@pytest.mark.parametrize("kind,n", [("families", 2000), ("erdos_renyi", 1500), ("stars", 800), ("dense", 150)])
def test_dendrogram_matches_scipy(method, kind, n):
    rng = np.random.default_rng([L.METHODS.index(method), n])
    n, a, b, ani = graph(kind, rng, n)
    check_scipy(n, a, b, ani, method, [0.905, 0.93, 0.955, 0.9712, 0.985])
