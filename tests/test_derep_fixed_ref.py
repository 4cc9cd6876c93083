"""tests/derep_fixed_ref.py (sk_dereplicate_fixed's waves) against tests/cluster_ref.py's greedy clusters of the triangle's
rows without the rows between two fixed genomes, on random pair oracles: every fixed-set size from none to all, wave sizes
1, 2, 7, 64, the library default and >= n, three thresholds.  rep, cluster and every member's joining pair equal; no pair
chained twice; no pair of two fixed genomes screened or chained (the restatement asserts it).  With an edge-free fixed set
(the representatives of an earlier run) it equals tests/derep_ref.py's plain waves, and with n_fixed = 0 it chains exactly
what they chain."""
import numpy as np
import pytest

import cluster_ref as R
import derep_fixed_ref as F
import derep_ref as D

WAVES = (1, 2, 7, 64, 0, 10_000)
THRESHOLDS = (0.95, 0.975, 0.99)


def random_case(rng, n):
    """screen-passing pairs in families plus random cross pairs; ANIs from a small set (ties) with sentinels"""
    fam = rng.integers(0, max(n // 6, 1), n)
    pairs = set()
    for i in range(n):
        for j in range(i + 1, n):
            if (fam[i] == fam[j] and rng.random() < 0.8) or rng.random() < 0.02:
                pairs.add((i, j))
    vals = np.array([0.96, 0.97, 0.975, 0.99, 0.999, 0.94, 0.5, 0.1, -1, np.nan], np.float32)
    ani = {p: vals[rng.integers(0, 6)] if fam[p[0]] == fam[p[1]] else vals[rng.integers(0, len(vals))] for p in sorted(pairs)}
    return pairs, ani


def fixed_sizes(n):
    return sorted({0, min(1, n), min(3, n), n // 2, max(n - 1, 0), n})


def expected(n, screen, ani, min_ani, rank, n_fixed):
    """cluster_ref's greedy clusters on the screen's rows without those joining two fixed genomes; the kept pair keys"""
    fixed = set(np.argsort(rank, kind="stable")[:n_fixed].tolist())
    keys = [p for p in sorted(screen) if not (p[0] in fixed and p[1] in fixed)]
    a = np.array([p[0] for p in keys], np.int64); b = np.array([p[1] for p in keys], np.int64)
    av = np.array([ani[p] for p in keys], np.float32)
    erep, ecl, eedge = R.greedy(n, a, b, av, min_ani, rank)
    return erep, ecl, eedge, keys, fixed


def check(n, screen, ani, min_ani, rank, n_fixed, wave):
    erep, ecl, eedge, keys, fixed = expected(n, screen, ani, min_ani, rank, n_fixed)
    rep, cl, join, chained, screened, waves = F.dereplicate(n, screen, ani, min_ani, rank, wave, n_fixed)
    assert np.array_equal(rep, erep) and np.array_equal(cl, ecl), (n, n_fixed, wave, min_ani)
    assert len(chained) == len(set(chained)) and screened >= len(chained)
    assert not any(p[0] in fixed and p[1] in fixed for p in chained)
    assert all(rep[g] == g and cl[g] == i for i, g in enumerate(np.argsort(rank, kind="stable")[:n_fixed]))
    for g in range(n):
        assert (join[g] is None) if erep[g] == g else join[g] == keys[int(eedge[g])]
    assert waves == len(F.wave_bounds(n, n_fixed, wave))
    if n_fixed == n:
        assert waves == 0 and screened == 0 and not chained
    return rep, cl, join, chained


@pytest.mark.parametrize("seed", range(30))
def test_fixed_waves_equal_greedy_without_fixed_pairs(seed):
    rng = np.random.default_rng(seed)
    n = int(rng.integers(1, 70))
    screen, ani = random_case(rng, n)
    rank = rng.permutation(n) if seed % 3 else np.arange(n)[::-1]
    for n_fixed in fixed_sizes(n):
        for min_ani in THRESHOLDS:
            for w in WAVES:
                check(n, screen, ani, min_ani, rank, n_fixed, w)


def test_fixed_sets_with_edges_inside_reached():
    """the random cases put edges inside the fixed set, where the fixed genomes stay representatives against the plain waves"""
    differs = 0
    for seed in range(30):
        rng = np.random.default_rng(seed)
        n = int(rng.integers(1, 70))
        screen, ani = random_case(rng, n)
        rank = rng.permutation(n) if seed % 3 else np.arange(n)[::-1]
        for n_fixed in fixed_sizes(n):
            rep = F.dereplicate(n, screen, ani, 0.95, rank, 7, n_fixed)[0]
            differs += not np.array_equal(rep, D.dereplicate(n, screen, ani, 0.95, rank, 7)[0])
    assert differs > 0


@pytest.mark.parametrize("seed", range(20))
def test_no_fixed_is_the_plain_waves(seed):
    rng = np.random.default_rng(100 + seed)
    n = int(rng.integers(1, 70))
    screen, ani = random_case(rng, n)
    rank = rng.permutation(n)
    for w in (1, 7, 10_000):
        rep, cl, join, chained = check(n, screen, ani, 0.975, rank, 0, w)
        drep, dcl, djoin, dchained = D.dereplicate(n, screen, ani, 0.975, rank, w)
        assert np.array_equal(rep, drep) and np.array_equal(cl, dcl) and join == djoin and chained == dchained


@pytest.mark.parametrize("seed", range(20))
def test_edge_free_fixed_set_equals_the_plain_waves(seed):
    """F = the representatives of an earlier run over the first genomes (edge-free), ranked first: the result is the plain
    waves' on the same ranks"""
    rng = np.random.default_rng(200 + seed)
    n = int(rng.integers(2, 70))
    screen, ani = random_case(rng, n)
    for min_ani in THRESHOLDS:
        old = int(rng.integers(1, n + 1))            # the earlier catalogue: genomes 0 .. old - 1
        sub = {p: ani[p] for p in screen if p[1] < old}
        orank = rng.permutation(old)
        orep = D.dereplicate(old, set(sub), sub, min_ani, orank, 7)[0]
        reps = [g for g in np.argsort(orank, kind="stable") if orep[g] == g]
        rest = [g for g in rng.permutation(n) if g not in set(reps)]
        rank = np.empty(n, np.int64)
        rank[np.array(reps + rest, np.int64)] = np.arange(n)
        for w in (1, 3, 0):
            rep, cl, join, _ = check(n, screen, ani, min_ani, rank, len(reps), w)
            drep, dcl, djoin, _ = D.dereplicate(n, screen, ani, min_ani, rank, w or 64)
            assert np.array_equal(rep, drep) and np.array_equal(cl, dcl) and join == djoin


def test_all_fixed_has_no_wave_and_no_pair():
    rng = np.random.default_rng(5)
    screen, ani = random_case(rng, 40)
    rep, cl, join, chained, screened, waves = F.dereplicate(40, screen, ani, 0.95, rng.permutation(40), 0, 40)
    assert waves == 0 and screened == 0 and chained == [] and np.array_equal(rep, np.arange(40))
