"""tests/derep_ref.py (sk_dereplicate's wave algorithm) against tests/cluster_ref.py's greedy clusters of the triangle's rows, on
random graphs at wave sizes 1, 2, 7, 64 and >= n: rep and cluster equal, every member joined by the row cluster_ref picks,
no pair chained twice and only pairs that pass the screen chained.  The graphs have ties in ANI, pairs that pass the screen
but are no edge (ANI below the threshold, NaN, -1, 0.1), isolated genomes, members whose best representative ranks after
them and representatives first met inside a wave; the test asserts that each of these occurred."""
import numpy as np
import pytest

import cluster_ref as R
import derep_ref as D

WAVES = (1, 2, 7, 64, 10_000)


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


def run_case(seed):
    """one random graph at every wave size and threshold; returns how often each edge case occurred"""
    rng = np.random.default_rng(seed)
    n = int(rng.integers(1, 90))
    screen, ani = random_case(rng, n)
    keys = sorted(screen)
    a = np.array([p[0] for p in keys], np.int64); b = np.array([p[1] for p in keys], np.int64)
    av = np.array([ani[p] for p in keys], np.float32)
    rank = rng.permutation(n) if seed % 3 else np.arange(n)[::-1]
    seen = {"late_rep": 0, "rep_in_wave": 0, "isolated": 0, "tie": 0}
    for min_ani in (0.95, 0.975, 0.99):
        erep, ecl, eedge = R.greedy(n, a, b, av, min_ani, rank)
        for w in WAVES:
            rep, cl, join, chained = D.dereplicate(n, screen, ani, min_ani, rank, w)
            assert np.array_equal(rep, erep) and np.array_equal(cl, ecl), (n, w, min_ani)
            assert len(chained) == len(set(chained))
            for g in range(n):
                if erep[g] == g:
                    assert join[g] is None
                    continue
                assert join[g] == keys[int(eedge[g])]
                if rank[erep[g]] > rank[g]:
                    seen["late_rep"] += 1
            if w == 7:      # a member whose representative was chosen in its own wave
                pos = np.empty(n, np.int64); pos[np.argsort(rank, kind="stable")] = np.arange(n)
                seen["rep_in_wave"] += int(sum(erep[g] != g and pos[g] // w == pos[erep[g]] // w for g in range(n)))
        deg = np.bincount(np.concatenate([a, b]), minlength=n) if len(a) else np.zeros(n, np.int64)
        seen["isolated"] += int((deg == 0).sum())
    _, counts = np.unique(av[np.isfinite(av)], return_counts=True)
    seen["tie"] += int((counts > 1).sum())
    return seen


@pytest.mark.parametrize("seed", range(40))
def test_waves_equal_greedy(seed):
    run_case(seed)


def test_cases_reached_their_edges():
    seen = {}
    for seed in range(40):
        for k, v in run_case(seed).items():
            seen[k] = seen.get(k, 0) + v
    assert all(v > 0 for v in seen.values()), seen


def test_fewer_pairs_than_the_triangle():
    """families of 20 ranked at random: the waves chain far fewer pairs than the triangle's screen passes"""
    rng = np.random.default_rng(99)
    n = 400
    fam = np.arange(n) // 20
    screen = {(i, j) for i in range(n) for j in range(i + 1, n) if fam[i] == fam[j]}
    ani = {p: np.float32(0.97 + 0.02 * rng.random()) for p in sorted(screen)}
    rank = rng.permutation(n)
    _, _, _, chained = D.dereplicate(n, screen, ani, 0.95, rank, 16)
    assert len(chained) * 4 < len(screen)
