"""sk_dereplicate_store (skani_b200.dereplicate_store) against sk_dereplicate on one in-memory set holding the same genomes
with the same name ranks: rep, cluster and every join row byte for byte, and the count fields of sk_derep_stats, every context
on GPU 0.  One and two contexts; wave sizes 1, 3 and the default; a derived budget (one working set per chain step), a budget
of about 1.05 x the largest family's bytes (many working sets) and about 0.45 x (components cut into chunk pairs), each case
checked through sk_store_stats.  Synthetic families in length, random and reverse rank order with contiguous and shuffled
genome ids, the E. coli goldens, viruses.fna per record with equal name ranks, genomes under 20 markers and without markers
at low and high indices with the rescue on and off, AF filters that make -1 sentinels, thresholds 0.8 / 0.95 / 0.99, one case
against sk_cluster on sk_triangle_store's rows, and every refusal."""
import ctypes as C
import os
import re

import numpy as np
import pytest

from bench_support import synth
from fasta_py import read_fastx

pytestmark = pytest.mark.gpu

GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
N, L, G = 40, 200_000, 5
WAVES = (1, 3, 0)
COUNTS = ("pairs_screened", "pairs_chained", "n_edges", "n_clusters", "waves", "rounds")


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


def store_of_genomes(sk, ctx, genomes, groups=3, ranks=None):
    """Genomes (lists of contigs) sketched in `groups` consecutive groups into a new store; name ranks set when given."""
    st = sk.SketchStore()
    bounds = np.linspace(0, len(genomes), groups + 1).astype(int)
    for a, b in zip(bounds[:-1], bounds[1:]):
        if a == b:
            continue
        s = sk.sketch_sequences(ctx, genomes[a:b])
        assert len(s) == b - a
        st.add(s)
        s.free()
    if ranks is not None:
        st.set_name_ranks(ranks)
    return st


def store_of_set(sk, s):
    """One store holding set s (its name ranks included: an empty store keeps them as they are)."""
    st = sk.SketchStore()
    st.add(s)
    return st


def length_rank(s):
    total = np.array([s.info(g)["total_len"] for g in range(len(s))], np.int64)
    order = np.lexsort((np.arange(len(s)), -total))
    rank = np.empty(len(s), np.uint32)
    rank[order] = np.arange(len(s))
    return rank


def ranks_for(order, s, seed=1):
    n = len(s)
    return {"length": length_rank(s), "random": np.random.default_rng(seed).permutation(n).astype(np.uint32),
            "reverse": np.arange(n, dtype=np.uint32)[::-1].copy()}[order]


def check(ctxs, s, st, rank, min_ani, mp, waves=WAVES, budget=0):
    """dereplicate_store == dereplicate on the in-memory set s at every wave size; returns the store stats per wave"""
    import skani_b200 as sk
    out = {}
    for w in waves:
        erep, ecl, ejoin, est = sk.dereplicate(ctxs[0], s, rank, min_ani=min_ani, mp=mp, wave=w)
        rep, cl, join, dst, sst = sk.dereplicate_store(ctxs, st, rank, min_ani=min_ani, mp=mp, wave=w, device_budget=budget)
        assert np.array_equal(rep, erep) and np.array_equal(cl, ecl), (w, np.nonzero((rep != erep) | (cl != ecl))[0][:5])
        assert join.tobytes() == ejoin.tobytes(), w
        for f in COUNTS:
            assert getattr(dst, f) == getattr(est, f), (w, f)
        assert (sst.n_working_sets > 0) == (dst.pairs_chained > 0) and sst.t_screen > 0
        assert budget == 0 or sst.max_working_set_bytes <= budget
        out[w] = (dst, sst)
    return out


# ---- synthetic families: contexts x budgets x ids ------------------------------------------------------------------------
@pytest.fixture(scope="module", params=["contiguous", "shuffled"])
def families(request, ctxs):
    import skani_b200 as sk
    ctx = ctxs[0]
    if request.param == "contiguous":
        bases, off, goc = synth.generate(0, N, L, G=G)
    else:
        bases, off, goc = synth.generate_ids(synth.shuffled_ids(N, 11), L, G=G)
    ranks = np.arange(N, dtype=np.uint64)
    s = sk.sketch_contigs(ctx, bases, off, goc, N)
    s.set_name_ranks(ranks)
    st = store_of_groups(sk, ctx, bases, off, goc, N, ranks=ranks)
    gb = np.array([st.genome_bytes(g) for g in range(N)])
    ids = np.array(synth.shuffled_ids(N, 11) if request.param == "shuffled" else np.arange(N), np.int64)
    family = max(gb[ids // G == f].sum() for f in range(N // G))   # the largest family's bytes
    yield sk, s, st, gb, family
    st.free()
    s.free()


BUDGETS = {"derived": None, "many_sets": 1.05, "chunk_pairs": 0.45}   # x the largest family's bytes


@pytest.mark.parametrize("n_ctx", [1, 2])
@pytest.mark.parametrize("case", sorted(BUDGETS))
def test_synthetic_families(ctxs, families, case, n_ctx, capfd, monkeypatch):
    sk, s, st, gb, family = families
    mult = BUDGETS[case]
    budget = 0 if mult is None else int(max(mult * family, 2 * gb.max() + 1))
    monkeypatch.setenv("SK_TRACE", "1")
    for order in ("length", "random", "reverse"):
        rank = ranks_for(order, s)
        capfd.readouterr()
        res = check(ctxs[:n_ctx], s, st, rank, 0.95, sk.map_params(), budget=budget)
        trace = [ln for ln in capfd.readouterr().err.splitlines() if ln.startswith("[sk_dereplicate_store]")]
        assert len(trace) == sum(sst.n_working_sets for _, sst in res.values())
        dst, sst = res[0]          # the default waves: one wave of every genome, so three chain steps at most
        steps = 2 * dst.waves + 1
        if case == "derived":      # one working set per chain step
            assert all(re.search(r"working set 1/1: ", ln) for ln in trace), trace[:3]
            assert sst.n_split_components == 0 and sst.n_working_sets <= steps
        elif case == "many_sets":
            assert sst.n_working_sets > steps and sst.n_split_components == 0
        else:
            assert sst.n_split_components > 0 and sst.n_working_sets > steps


def test_thresholds(ctxs, families):
    sk, s, st, gb, family = families
    rank = ranks_for("random", s, seed=5)
    for t in (0.8, 0.95, 0.99):
        check(ctxs, s, st, rank, t, sk.map_params(), budget=int(1.05 * family))


def test_cluster_on_triangle_store_rows(ctxs, families):
    """the store path also equals sk_cluster (greedy) on sk_triangle_store's rows"""
    sk, s, st, gb, family = families
    rank = ranks_for("length", s)
    tri, _ = sk.triangle_store(ctxs, st, device_budget=int(1.05 * family))
    erep, ecl, eedge, _ = sk.cluster(ctxs[0], N, tri, rank, min_ani=0.95)
    rep, cl, join, _, _ = sk.dereplicate_store(ctxs, st, rank, min_ani=0.95, wave=3, device_budget=int(max(0.45 * family, 2 * gb.max() + 1)))
    mem = erep != np.arange(N)
    assert mem.any() and np.array_equal(rep, erep) and np.array_equal(cl, ecl)
    assert join[mem].tobytes() == tri[eedge[mem].astype(np.int64)].tobytes()


# ---- real genomes ---------------------------------------------------------------------------------------------------------
def _ecoli():
    return [[seq for _, seq in read_fastx(os.path.join(GOLD, f))] for f in ("e.coli-EC590.fasta.gz", "e.coli-K12.fasta.gz")]


def test_ecoli_goldens(ctxs):
    import skani_b200 as sk
    genomes = _ecoli()
    s = sk.sketch_sequences(ctxs[0], genomes)
    st = store_of_genomes(sk, ctxs[0], genomes, groups=2, ranks=[0, 1])
    s.set_name_ranks([0, 1])
    for rank in ([0, 1], [1, 0]):
        for t in (0.95, 0.99, 0.999):
            check(ctxs, s, st, np.array(rank, np.uint32), t, sk.map_params())
    st.free()
    # -i: every record its own sketch, records of one file sharing a name rank
    vir = [seq for _, seq in read_fastx(os.path.join(GOLD, "viruses.fna"))]
    si = sk.sketch_sequences(ctxs[0], genomes + [vir], individual_contig=True)
    assert len(si) > 3
    sti = store_of_set(sk, si)
    gb = max(sti.genome_bytes(g) for g in range(len(si)))
    for t in (0.8, 0.95):
        check(ctxs, si, sti, length_rank(si), t, sk.map_params(learned_ani=False))
        check(ctxs, si, sti, length_rank(si), t, sk.map_params(learned_ani=False), waves=(0,), budget=int(2.2 * gb))
    sti.free()


def test_viruses_individual(ctxs):
    import skani_b200 as sk
    recs = [seq for _, seq in read_fastx(os.path.join(GOLD, "viruses.fna"))]
    s = sk.sketch_sequences(ctxs[0], [recs], individual_contig=True)
    assert sum(s.info(g)["n_markers"] < 20 for g in range(len(s))) > 0
    st = store_of_set(sk, s)
    gb = max(st.genome_bytes(g) for g in range(len(s)))
    for rescue in (True, False):
        for t in (0.8, 0.95):
            mp = sk.map_params(rescue_small=rescue, learned_ani=False)
            check(ctxs, s, st, length_rank(s), t, mp)
            check(ctxs, s, st, length_rank(s), t, mp, waves=(0,), budget=int(2.2 * gb))
    st.free()


def small_and_empty_genomes():
    """families of 100 kbp genomes plus slices of family members of 3-25 kbp (about 3-25 markers) and poly-A genomes without
    markers, at the lowest and highest genome indices"""
    bases, off, goc = synth.generate(0, 60, 100_000, G=10)
    fam = [[bytes(bases[int(off[i]):int(off[i + 1])]) for i in np.nonzero(goc == g)[0]] for g in range(60)]
    rng = np.random.default_rng(7)
    small = []
    for k in range(24):
        src = b"".join(fam[int(rng.integers(60))])
        ln = int(rng.choice([3_000, 12_000, 18_000, 19_500, 20_500, 25_000]))
        a = int(rng.integers(0, len(src) - ln))
        small.append([src[a:a + ln]])
    empty = [[b"A" * 800]]
    return small[:12] + empty + fam + empty + small[12:]


@pytest.fixture(scope="module")
def small_and_empty(ctxs):
    import skani_b200 as sk
    genomes = small_and_empty_genomes()
    n = len(genomes)
    s = sk.sketch_sequences(ctxs[0], genomes)
    s.set_name_ranks(np.arange(n))
    cards = [s.info(g)["n_markers"] for g in range(n)]
    assert min(cards) == 0 and any(0 < c < 20 for c in cards[:12]) and any(0 < c < 20 for c in cards[-12:])
    st = store_of_genomes(sk, ctxs[0], genomes, ranks=np.arange(n))
    assert st.n_genomes() == n
    yield sk, s, st
    st.free()
    s.free()


@pytest.mark.parametrize("rescue", [True, False])
def test_small_and_empty_genomes(ctxs, small_and_empty, rescue):
    sk, s, st = small_and_empty
    n = len(s)
    lr = length_rank(s)
    gb = max(st.genome_bytes(g) for g in range(n))
    rng = np.random.default_rng(3)
    for rank in (lr, (n - 1 - lr).astype(np.uint32), rng.permutation(n).astype(np.uint32)):   # small genomes last, first, anywhere
        for t in (0.8, 0.95):
            check(ctxs, s, st, rank, t, sk.map_params(rescue_small=rescue), waves=(1, 0))
        check(ctxs, s, st, rank, 0.95, sk.map_params(rescue_small=rescue), waves=(3,), budget=int(4.5 * gb))


def test_af_filters_make_sentinels(ctxs, small_and_empty):
    sk, s, st = small_and_empty
    for mp in (sk.map_params(min_af=0.5), sk.map_params(both_min_af=0.5)):
        pairs = sk.screen_triangle(ctxs[0], s, mp)
        assert (sk.chain_pairs(ctxs[0], s, s, pairs, mp, as_array=True)["ani"] == -1).any()
        check(ctxs, s, st, length_rank(s), 0.95, mp)


# ---- edges and refusals ---------------------------------------------------------------------------------------------------
def test_empty_and_single(ctxs):
    import skani_b200 as sk
    st = sk.SketchStore()
    rep, cl, join, dst, sst = sk.dereplicate_store(ctxs, st, np.zeros(0, np.uint32))
    assert len(rep) == len(cl) == len(join) == 0 and dst.n_clusters == 0 and dst.waves == 0 and sst.n_working_sets == 0
    s = sk.sketch_sequences(ctxs[0], [[b"ACGT" * 5000]])
    st.add(s)
    rep, cl, join, dst, sst = sk.dereplicate_store(ctxs, st, np.zeros(1, np.uint32))
    erep, ecl, ejoin, est = sk.dereplicate(ctxs[0], s, np.zeros(1, np.uint32))
    assert rep.tolist() == [0] and cl.tolist() == [0] and join.tobytes() == ejoin.tobytes()
    assert dst.n_clusters == 1 and dst.pairs_chained == 0 and sst.n_working_sets == 0
    st.free()


def test_refusals(ctxs):
    import skani_b200 as sk
    from skani_b200 import _lib
    ctx = ctxs[0]
    n = 6
    bases, off, goc = synth.generate(0, n, 60_000, G=3)
    s = sk.sketch_contigs(ctx, bases, off, goc, n)
    s.set_name_ranks(np.arange(n))
    st = store_of_groups(sk, ctx, bases, off, goc, n, groups=2, ranks=np.arange(n))
    rank = np.arange(n, dtype=np.uint32)
    for bad, msg in ((np.array([0, 0, 1, 2, 3, 4], np.uint32), "permutation"), (np.array([0, 1, 2, 3, 4, 6], np.uint32), "permutation")):
        with pytest.raises(sk.host.SkaniError, match=r"rc=-2.*" + msg):
            sk.dereplicate_store(ctxs, st, bad)
    with pytest.raises(sk.host.SkaniError, match=r"rc=-2.*NaN"):
        sk.dereplicate_store(ctxs, st, rank, min_ani=float("nan"))
    with pytest.raises(sk.host.SkaniError, match=r"rc=-2.*appears twice"):
        sk.dereplicate_store([ctx, ctxs[1], ctx], st, rank)
    # a genome over budget / 2: SK_ERR_NOMEM before any device work
    gb = max(st.genome_bytes(g) for g in range(n))
    before = [c.launches for c in ctxs]
    with pytest.raises(sk.host.SkaniError, match=r"rc=-3.*more than half the working-set budget"):
        sk.dereplicate_store(ctxs, st, rank, device_budget=gb)
    assert [c.launches for c in ctxs] == before
    # NULL in every pointer argument
    mp, dp, dst, sst = sk.map_params(), _lib.DerepParams(0.95, 0), _lib.DerepStats(), _lib.StoreStats()
    o32 = np.zeros(n, np.uint32); join = np.zeros(n, sk.host.RESULT_DTYPE)
    hs = (C.c_void_p * 2)(*[c.h for c in ctxs])
    args = [hs, 2, st.h, C.byref(mp), rank.ctypes.data, C.byref(dp), 0, o32.ctypes.data, o32.ctypes.data, join.ctypes.data, C.byref(dst), C.byref(sst)]
    for i in (2, 3, 4, 5, 7, 8, 9):
        bad = list(args)
        bad[i] = None
        assert ctx.L.sk_dereplicate_store(*bad) == -2, i
        assert "NULL" in ctx.L.sk_last_error(ctx.h).decode(), i
    bad = list(args)
    bad[0] = None
    assert ctx.L.sk_dereplicate_store(*bad) == -2
    bad = list(args)
    bad[1] = 0
    assert ctx.L.sk_dereplicate_store(*bad) == -2
    nulls = (C.c_void_p * 2)(ctx.h, None)
    bad = list(args)
    bad[0] = nulls
    assert ctx.L.sk_dereplicate_store(*bad) == -2 and "NULL context" in ctx.L.sk_last_error(ctx.h).decode()
    assert ctx.L.sk_dereplicate_store(*args[:10], None, None) == 0       # the stats may be NULL
    # the contexts still work after every refusal
    check(ctxs, s, st, rank, 0.95, mp)
    check(ctxs[1:], s, st, rank, 0.95, mp, waves=(0,))
    st.free()
    s.free()
