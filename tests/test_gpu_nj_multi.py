"""sk_neighbor_joining_multi (skani_b200.neighbor_joining_multi): the distance matrix split over 1 to 4 contexts gives the
join table of sk_neighbor_joining byte for byte, and tests/nj_ref.py's where the reference is fast enough.  Sizes around the
scan tile and the compactions (bands that empty as the square shrinks, more contexts than row tiles), random sparse graphs,
all pairs missing, families with one ANI and additive trees recovered exactly; the stats; the refusals on ctxs[0]; and
`tree --gpus 2 | 3` byte-identical to `tree` on FASTA inputs and on a sketch database (the store path, also with a small
device budget), with -i labels."""
import numpy as np
import pytest

import cluster_ref as CR
import nj_ref as N
from test_gpu_cli_cluster import VIR, run
from test_gpu_cli_cluster import synth_files  # noqa: F401  (fixture)

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def ctxs():
    """four contexts on device 0"""
    import skani_b200 as sk
    cs = [sk.Context(0) for _ in range(4)]
    yield cs
    for c in cs:
        c.close()


def same(got, want, n):
    assert np.array_equal(got["a"], want["a"]) and np.array_equal(got["b"], want["b"]), n
    assert np.array_equal(got["len_a"].view(np.uint64), want["len_a"].view(np.uint64)), n
    assert np.array_equal(got["len_b"].view(np.uint64), want["len_b"].view(np.uint64)), n


def check(cs, n, a, b, ani, ref=True, counts=(1, 2, 3, 4)):
    import skani_b200 as sk
    res = CR.as_results(a, b, ani)
    base, st = sk.neighbor_joining(cs[0], n, res)
    if ref:
        same(base, N.nj_results(n, a, b, ani), n)
    for k in counts:
        joins, st2 = sk.neighbor_joining_multi(cs[:k], n, res)
        assert joins.tobytes() == base.tobytes(), (n, k)
        assert (st2.n_edges, st2.joins, st2.compactions) == (st.n_edges, st.joins, st.compactions), (n, k)
    return st


# 86: the first compaction leaves one row tile (three of four bands empty); 256: four bands of one tile, then three tiles
@pytest.mark.parametrize("n", [2, 3, 4, 63, 64, 65, 86, 128, 129, 256, 300, 700])
def test_sizes_around_tile_and_compaction(ctxs, n):
    rng = np.random.default_rng(n)
    st = check(ctxs, *CR.erdos_renyi(rng, n, 4 * n))
    assert n < 100 or st.compactions > 0


@pytest.mark.parametrize("seed", range(2))
def test_random_sparse(ctxs, seed):
    rng = np.random.default_rng(2000 + seed)
    n = [900, 1500][seed]
    if seed % 2:
        check(ctxs, *CR.families(rng, n, int(rng.integers(3, 12)), 2 * n))
    else:
        check(ctxs, *CR.erdos_renyi(rng, n, 5 * n))


@pytest.mark.parametrize("n", [2, 3, 65, 200])
def test_all_missing(ctxs, n):
    empty = np.zeros(0, np.uint32)
    check(ctxs, n, empty, empty, np.zeros(0, np.float32))


@pytest.mark.parametrize("n", [130, 400])
def test_families_with_one_ani(ctxs, n):
    rng = np.random.default_rng(n)
    n, a, b, ani = CR.families(rng, n, 5, n // 2)
    check(ctxs, n, a, b, np.full(len(a), np.float32(0.97)))


@pytest.mark.parametrize("n", [500, 3000])
def test_additive_trees_recovered(ctxs, n):
    import skani_b200 as sk
    rng = np.random.default_rng(n)
    D, parent, _ = N.random_additive(rng, n)
    a, b = np.triu_indices(n, 1)
    a, b = a.astype(np.uint32), b.astype(np.uint32)
    ani = (1.0 - D[a, b]).astype(np.float32)
    st = check(ctxs, n, a, b, ani, ref=False, counts=(2, 3))
    joins, _ = sk.neighbor_joining_multi(ctxs[:3], n, CR.as_results(a, b, ani))
    parent2, length2 = N.tree_of_joins(n, joins)
    assert N.splits(n, parent2) == N.splits(n, parent)
    assert np.array_equal(N.patristic(n, parent2, length2), D)
    assert st.compactions >= 4


def test_distinct_devices():
    import torch
    import skani_b200 as sk
    k = min(torch.cuda.device_count(), 4)
    if k < 2:
        pytest.skip("one CUDA device")
    cs = [sk.Context(d) for d in range(k)]
    try:
        rng = np.random.default_rng(7)
        for n in (65, 129, 700):
            check(cs, *CR.erdos_renyi(rng, n, 4 * n), counts=range(2, k + 1))
    finally:
        for c in cs:
            c.close()


def test_refusals(ctxs):
    import skani_b200 as sk
    from skani_b200.host import SkaniError

    def refused(cs, n, a, b, ani, *texts):
        with pytest.raises(SkaniError) as e:
            sk.neighbor_joining_multi(cs, n, CR.as_results(np.array(a, np.uint32), np.array(b, np.uint32), np.array(ani, np.float32)))
        assert all(t in str(e.value) for t in texts), str(e.value)
    two = ctxs[:2]
    refused(two, 3, [0, 1], [1, 2], [0.9, 1.0001], "sk_neighbor_joining", "ani > 1")
    refused(two, 3, [0, 1], [1, 3], [0.9, 0.9], "sk_neighbor_joining", "genome id")
    refused(two, 3, [0, 2], [1, 2], [0.9, 0.9], "sk_neighbor_joining", "self pair")
    refused([ctxs[0], None], 3, [0], [1], [0.9], "context 1: NULL context")
    refused([ctxs[0], ctxs[1], ctxs[0]], 3, [0], [1], [0.9], "context 2: the same context appears twice")
    for n in (0, 1):
        joins, st = sk.neighbor_joining_multi(two, n, CR.as_results([], [], []))
        assert len(joins) == 0 and st.joins == 0


@pytest.mark.parametrize("gpus", ["2", "3"])
def test_cli_identical(synth_files, tmp_path, gpus):  # noqa: F811
    from test_gpu_cli_cluster import EC, K12
    inputs = synth_files + [EC, K12, VIR]
    base, err = run(["tree"] + inputs)
    assert "contexts" not in err.split("tree by nj", 1)[1].split("\n")[0]
    out, err = run(["tree", "--gpus", gpus] + inputs)
    assert out == base and "tree by nj (" in err and ") on %s contexts," % gpus in err, err
    db = str(tmp_path / "db")
    run(["sketch"] + inputs + ["-o", db])
    assert run(["tree", db])[0] == base
    for env in (None, {"SK_DEVICE_BUDGET_MB": "8"}):   # a database on several GPUs takes the store path
        out, err = run(["tree", "--gpus", gpus, db], env)
        assert out == base and "Store path" in err and ") on %s contexts," % gpus in err, err
    ind = run(["tree", "-i", VIR])[0]
    assert run(["tree", "-i", "--gpus", gpus, VIR])[0] == ind
