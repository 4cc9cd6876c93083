"""tests/nj_ref.py, the exact reference of sk_neighbor_joining, on the CPU: it recovers random additive trees with patristic
distances equal to the input bit for bit; on random tie-free matrices it gives the textbook algorithm's topology and branch
lengths; hand-checked n = 2, 3 and 4; the all-missing graph, where the join order is the tie rule alone; and the Newick
parser on quoting and a deep caterpillar."""
import numpy as np
import pytest

import nj_ref as N


def joined_patristic(n, joins):
    parent, length = N.tree_of_joins(n, joins)
    return N.patristic(n, parent, length)


@pytest.mark.parametrize("seed", range(12))
def test_additive_trees_recovered_exactly(seed):
    rng = np.random.default_rng(seed)
    n = int(rng.integers(3, 200 if seed % 3 == 0 else 60))
    D, parent, _ = N.random_additive(rng, n)
    ani = (1.0 - D).astype(np.float32)
    assert np.array_equal(1.0 - ani.astype(np.float64), D)        # the float32 round trip is exact
    a, b = np.triu_indices(n, 1)
    joins = N.nj_results(n, a, b, ani[a, b])
    assert np.array_equal(joined_patristic(n, joins), D)
    assert N.splits(n, N.tree_of_joins(n, joins)[0]) == N.splits(n, parent)


@pytest.mark.parametrize("seed", range(8))
def test_tie_free_matches_textbook(seed):
    rng = np.random.default_rng(100 + seed)
    n = int(rng.integers(3, 30))
    D = rng.random((n, n)) * 0.5 + 0.2
    D = np.triu(D, 1)
    D = D + D.T
    got = N.nj(D)
    want = N.nj_textbook(D)
    assert len(got) == len(want) == n - 1
    # at m = 4 the complementary pairs have equal Q and at m = 3 all three do, so the last three rows follow rounding and the
    # tie rule; the unrooted tree is the same
    wt = np.zeros(n - 1, N.NJ_JOIN_DTYPE)
    wt[:] = want
    assert np.allclose(joined_patristic(n, got), joined_patristic(n, wt), rtol=0, atol=1e-9)
    for r, (a, b, la, lb) in zip(got[:max(n - 4, 0)], want):
        if (int(r["a"]), int(r["b"])) == (a, b):
            assert abs(r["len_a"] - la) < 1e-9 and abs(r["len_b"] - lb) < 1e-9
        else:
            assert (int(r["a"]), int(r["b"])) == (b, a)
            assert abs(r["len_a"] - lb) < 1e-9 and abs(r["len_b"] - la) < 1e-9


def rows(j):
    return [(int(r["a"]), int(r["b"]), float(r["len_a"]), float(r["len_b"])) for r in j]


def test_small_by_hand():
    assert len(N.nj(np.zeros((0, 0)))) == 0 and len(N.nj(np.zeros((1, 1)))) == 0
    assert rows(N.nj([[0, 0.5], [0.5, 0]])) == [(0, 1, 0.25, 0.25)]
    # n = 3: every Q is d01 - R_0 - R_1 = -1.375 exactly; the tie goes to (0, 1).  R = (0.75, 0.875, 1.125),
    # delta_0 = 0.125 + (0.75 - 0.875) / 2, d_u2 = 0.5 (0.5 + 0.625 - 0.25)
    D = [[0, 0.25, 0.5], [0.25, 0, 0.625], [0.5, 0.625, 0]]
    assert rows(N.nj(D)) == [(0, 1, 0.0625, 0.1875), (3, 2, 0.21875, 0.21875)]
    # n = 4, the additive quartet ((0:1/8, 1:1/4):3/8, (2:1/16, 3:5/16)): Q(0,1) = Q(2,3) = -3 is the minimum, tie to (0, 1);
    # then m = 3 ties again, to (4, 2), and node 5 keeps id 0, so the last row is (5, 3)
    D = np.array([[0, .375, .5625, .8125], [.375, 0, .6875, .9375], [.5625, .6875, 0, .375], [.8125, .9375, .375, 0]])
    assert rows(N.nj(D)) == [(0, 1, 0.125, 0.25), (4, 2, 0.375, 0.0625), (5, 3, 0.15625, 0.15625)]
    assert np.array_equal(joined_patristic(4, N.nj(D)), D)


def test_all_missing_follows_tie_rule():
    n = 7
    j = N.nj_results(n, [], [], [])
    # every Q ties at every step, so (0, 1) joins first and the new node keeps slot 0: 0 with 1, then the result with 2, ...
    assert [(int(r["a"]), int(r["b"])) for r in j] == [(0, 1)] + [(n + t - 1, t + 1) for t in range(1, n - 1)]
    assert np.allclose(joined_patristic(n, j)[np.triu_indices(n, 1)], 1.0)


def test_newick_parser():
    labels, parent, length = N.parse_newick("(A:1,'b c':2,('it''s':0.5,D:1.5):3);")
    assert labels == ["A", "b c", "it's", "D"]
    P = N.patristic(4, parent, length)
    assert P[0, 1] == 3 and P[2, 3] == 2 and P[0, 2] == 4.5 and P[1, 3] == 6.5
    n = 5000                                    # a caterpillar nests n deep
    s = "L0:1"
    for k in range(1, n):
        s = "(%s,L%d:1):1" % (s, k)
    labels, parent, _ = N.parse_newick(s + ";")
    assert len(labels) == n and sum(p < 0 for p in parent) == 1
