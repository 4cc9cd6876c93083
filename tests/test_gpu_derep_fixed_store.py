"""sk_dereplicate_store_fixed (skani_b200.dereplicate_store_fixed) against sk_dereplicate_fixed on one in-memory set holding
the same genomes with the same name ranks: rep, cluster and every join row byte for byte, and the count fields of
sk_derep_stats.  One and two contexts on GPU 0; wave sizes 1, 3 and the default; a derived budget, about 1.05 x the largest
family's bytes (many working sets) and about 0.45 x (components cut into chunk pairs), each confirmed through
sk_store_stats; fixed sets spread over the store's three groups, of every size from none to all; n_fixed = 0 equal to
sk_dereplicate_store; the refusal of n_fixed > n_genomes."""
import numpy as np
import pytest

from bench_support import synth

pytestmark = pytest.mark.gpu

N, L, G = 40, 200_000, 5
WAVES = (1, 3, 0)
COUNTS = ("pairs_screened", "pairs_chained", "n_edges", "n_clusters", "waves", "rounds")
BUDGETS = {"derived": None, "many_sets": 1.05, "chunk_pairs": 0.45}   # x the largest family's bytes


@pytest.fixture(scope="module")
def ctxs():
    import skani_b200 as sk
    cs = [sk.Context(0), sk.Context(0)]
    yield cs
    for c in cs:
        c.close()


def store_of_groups(sk, ctx, bases, off, goc, n, groups=3, ranks=None):
    """The genomes sketched in `groups` consecutive groups, each added to a new store and freed; name ranks set when given."""
    st = sk.SketchStore()
    bounds = np.linspace(0, n, groups + 1).astype(int)
    for a, b in zip(bounds[:-1], bounds[1:]):
        idx = np.nonzero((goc >= a) & (goc < b))[0]
        lo, hi = int(off[idx[0]]), int(off[idx[-1] + 1])
        s = sk.sketch_contigs(ctx, bases[lo:hi], off[idx[0]:idx[-1] + 2] - off[idx[0]], goc[idx] - a, b - a)
        st.add(s)
        s.free()
    if ranks is not None:
        st.set_name_ranks(ranks)
    return st


@pytest.fixture(scope="module", params=["contiguous", "shuffled"])
def families(request, ctxs):
    import skani_b200 as sk
    ctx = ctxs[0]
    shuffled = request.param == "shuffled"
    bases, off, goc = synth.generate_ids(synth.shuffled_ids(N, 11), L, G=G) if shuffled else synth.generate(0, N, L, G=G)
    ranks = np.arange(N, dtype=np.uint64)
    s = sk.sketch_contigs(ctx, bases, off, goc, N)
    s.set_name_ranks(ranks)
    st = store_of_groups(sk, ctx, bases, off, goc, N, ranks=ranks)
    gb = np.array([st.genome_bytes(g) for g in range(N)])
    ids = np.array(synth.shuffled_ids(N, 11) if shuffled else np.arange(N), np.int64)
    family = max(gb[ids // G == f].sum() for f in range(N // G))   # the largest family's bytes
    yield sk, s, st, gb, family
    st.free()
    s.free()


def spread_rank(n, seed):
    """a random rank whose genomes alternate between the store's three groups, so that every fixed set of three or more genomes
    spreads over all of them"""
    rng = np.random.default_rng(seed)
    perm = [rng.permutation(gr) for gr in np.array_split(np.arange(n), 3)]
    first = [int(p[k]) for k in range(max(len(p) for p in perm)) for p in perm if k < len(p)]
    rank = np.empty(n, np.uint32)
    rank[np.array(first, np.int64)] = np.arange(n, dtype=np.uint32)
    return rank


def check(ctxs, s, st, rank, n_fixed, min_ani, mp, budget=0, waves=WAVES):
    """dereplicate_store_fixed == dereplicate_fixed on the in-memory set s at every wave size; the store stats per wave"""
    import skani_b200 as sk
    out = {}
    for w in waves:
        erep, ecl, ejoin, est = sk.dereplicate_fixed(ctxs[0], s, rank, n_fixed, min_ani=min_ani, mp=mp, wave=w)
        rep, cl, join, dst, sst = sk.dereplicate_store_fixed(ctxs, st, rank, n_fixed, min_ani=min_ani, mp=mp, wave=w, device_budget=budget)
        assert np.array_equal(rep, erep) and np.array_equal(cl, ecl), (n_fixed, w, np.nonzero((rep != erep) | (cl != ecl))[0][:5])
        assert join.tobytes() == ejoin.tobytes(), (n_fixed, w)
        for f in COUNTS:
            assert getattr(dst, f) == getattr(est, f), (n_fixed, w, f)
        assert (sst.n_working_sets > 0) == (dst.pairs_chained > 0)
        assert budget == 0 or sst.max_working_set_bytes <= budget
        out[w] = (dst, sst)
    return out


@pytest.mark.parametrize("n_ctx", [1, 2])
@pytest.mark.parametrize("case", sorted(BUDGETS))
def test_store_equals_in_memory(ctxs, families, n_ctx, case):
    sk, s, st, gb, family = families
    mult = BUDGETS[case]
    budget = 0 if mult is None else int(max(mult * family, 2 * gb.max() + 1))
    mp = sk.map_params()
    rank = spread_rank(N, 4)
    steps = split = 0
    for n_fixed in (0, 1, 7, N // 2, N - 1, N):
        for w, (dst, sst) in check(ctxs[:n_ctx], s, st, rank, n_fixed, 0.95, mp, budget).items():
            steps = max(steps, sst.n_working_sets - (2 * dst.waves + 1))   # > 0: more working sets than chain steps
            split += sst.n_split_components
            if n_fixed == N:
                assert dst.waves == 0 and dst.pairs_screened == 0 and sst.n_working_sets == 0
    assert (steps > 0) == (case != "derived") and (split > 0) == (case == "chunk_pairs")


def test_no_fixed_is_dereplicate_store(ctxs, families):
    sk, s, st, gb, family = families
    mp = sk.map_params()
    rank = spread_rank(N, 9)
    budget = int(1.05 * family)
    for w in WAVES:
        exp = sk.dereplicate_store(ctxs, st, rank, min_ani=0.95, mp=mp, wave=w, device_budget=budget)
        got = sk.dereplicate_store_fixed(ctxs, st, rank, 0, min_ani=0.95, mp=mp, wave=w, device_budget=budget)
        for a, b in zip(got[:3], exp[:3]):
            assert a.tobytes() == b.tobytes(), w
        for f in COUNTS:
            assert getattr(got[3], f) == getattr(exp[3], f), (w, f)
        assert got[4].n_working_sets == exp[4].n_working_sets and got[4].gathered_bytes == exp[4].gathered_bytes


def test_refusals(ctxs, families):
    sk, s, st, gb, family = families
    with pytest.raises(sk.host.SkaniError, match="sk_dereplicate_store_fixed: n_fixed = 41 fixed representatives, more than the 40 genomes"):
        sk.dereplicate_store_fixed(ctxs, st, np.arange(N, dtype=np.uint32), N + 1)
    check(ctxs, s, st, np.arange(N, dtype=np.uint32), 3, 0.95, sk.map_params(), waves=(0,))   # the contexts still work
