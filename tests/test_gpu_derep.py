"""sk_dereplicate (skani_b200.dereplicate) against sk_cluster's greedy clusters of the same set's triangle rows
(screen_triangle + chain_pairs): rep and cluster equal, and the row joining every member to its representative byte for
byte the row sk_cluster's edge points to.  Synthetic families, the E. coli goldens, per-record (-i) sets with equal name
ranks, genomes under 20 markers and without markers at low and high indices and ranks with the rescue on and off, AF
filters that turn chained rows into the -1 sentinel, thresholds 0.8 / 0.95 / 0.99, wave sizes 1, 3, 64, the default and
>= n; every refusal."""
import os

import numpy as np
import pytest

from bench_support import synth
from fasta_py import read_fastx

pytestmark = pytest.mark.gpu

GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
WAVES = (1, 3, 64, 0, 1 << 20)


@pytest.fixture(scope="module")
def ctx():
    import skani_b200 as sk
    c = sk.Context(0)
    yield c
    c.close()


def triangle_rows(ctx, s, mp):
    import skani_b200 as sk
    pairs = sk.screen_triangle(ctx, s, mp)
    return sk.chain_pairs(ctx, s, s, pairs, mp, as_array=True)


def check(ctx, s, rank, min_ani, mp, waves=WAVES):
    """dereplicate at every wave size equals cluster (greedy) on the triangle's rows; returns (last stats, triangle pairs)"""
    import skani_b200 as sk
    n = len(s)
    tri = triangle_rows(ctx, s, mp)
    erep, ecl, eedge, _ = sk.cluster(ctx, n, tri, rank, min_ani=min_ani)
    g = np.arange(n)
    mem = erep != g
    for w in waves:
        rep, cl, join, st = sk.dereplicate(ctx, s, rank, min_ani=min_ani, mp=mp, wave=w)
        assert np.array_equal(rep, erep) and np.array_equal(cl, ecl), (w, np.nonzero((rep != erep) | (cl != ecl))[0][:5])
        assert join[mem].tobytes() == tri[eedge[mem].astype(np.int64)].tobytes(), w
        assert np.isnan(join["ani"][~mem]).all()
        assert np.array_equal(join["ref_id"][~mem], g[~mem]) and np.array_equal(join["query_id"][~mem], g[~mem])
        assert st.n_clusters == int((~mem).sum())
        assert st.pairs_chained <= st.pairs_screened
        if w:
            assert st.waves == -(-n // w)
    return st, len(tri)


def length_rank(s):
    total = np.array([s.info(g)["total_len"] for g in range(len(s))], np.int64)
    order = np.lexsort((np.arange(len(s)), -total))
    rank = np.empty(len(s), np.uint32)
    rank[order] = np.arange(len(s))
    return rank


def family_set(ctx, n, L, G, seed=0):
    import skani_b200 as sk
    bases, off, goc = synth.generate(seed, seed + n, L, G=G)
    return sk.sketch_contigs(ctx, bases, off, goc, n), bases, off, goc


@pytest.mark.parametrize("order", ["length", "random", "reverse"])
def test_synthetic_families(ctx, order):
    import skani_b200 as sk
    s, *_ = family_set(ctx, 160, 100_000, 20)
    rng = np.random.default_rng(1)
    rank = {"length": length_rank(s), "random": rng.permutation(len(s)).astype(np.uint32),
            "reverse": np.arange(len(s), dtype=np.uint32)[::-1].copy()}[order]
    for t in (0.8, 0.95, 0.99):
        check(ctx, s, rank, t, sk.map_params())


def test_chains_far_fewer_pairs_than_the_triangle(ctx):
    """families of 30 scattered over the genome indices, as bench.py lays them out (equal lengths: rank = index order), at an
    ANI threshold that keeps most families whole (members differ by up to 5 % substitutions each from their ancestor)"""
    import skani_b200 as sk
    bases, off, goc = synth.generate_ids(synth.shuffled_ids(600, 5), 60_000, G=30)
    s = sk.sketch_contigs(ctx, bases, off, goc, 600)
    st, n_tri = check(ctx, s, length_rank(s), 0.9, sk.map_params(), waves=(32, 0))   # st: the default waves
    st32 = sk.dereplicate(ctx, s, length_rank(s), min_ani=0.9, mp=sk.map_params(), wave=32)[3]
    print("600 genomes in families of 30: triangle chains %d pairs, dereplicate %d with the default waves, %d with waves of 32 "
          "(%d clusters)" % (n_tri, st.pairs_chained, st32.pairs_chained, st.n_clusters))
    assert st32.pairs_chained * 3 < n_tri and st.pairs_chained * 3 < n_tri


def _ecoli():
    return [[seq for _, seq in read_fastx(os.path.join(GOLD, f))] for f in ("e.coli-EC590.fasta.gz", "e.coli-K12.fasta.gz")]


def test_ecoli_goldens(ctx):
    import skani_b200 as sk
    genomes = _ecoli()
    s = sk.sketch_sequences(ctx, genomes)
    for rank in ([0, 1], [1, 0]):
        for t in (0.95, 0.99, 0.999):
            check(ctx, s, np.array(rank, np.uint32), t, sk.map_params())
    # -i: every record its own sketch, records of one file sharing a name rank
    vir = [seq for _, seq in read_fastx(os.path.join(GOLD, "viruses.fna"))]
    si = sk.sketch_sequences(ctx, genomes + [vir], individual_contig=True)
    assert len(si) > 3
    for t in (0.8, 0.95):
        check(ctx, si, length_rank(si), t, sk.map_params(learned_ani=False))


def test_viruses_individual(ctx):
    import skani_b200 as sk
    recs = [seq for _, seq in read_fastx(os.path.join(GOLD, "viruses.fna"))]
    s = sk.sketch_sequences(ctx, [recs], individual_contig=True)
    small = sum(s.info(g)["n_markers"] < 20 for g in range(len(s)))
    assert small > 0
    for rescue in (True, False):
        for t in (0.8, 0.95):
            check(ctx, s, length_rank(s), t, sk.map_params(rescue_small=rescue, learned_ani=False))


def small_and_empty_set(ctx):
    """families of 100 kbp genomes plus slices of family members of 3-25 kbp (about 3-25 markers) and poly-A genomes without
    markers, at the lowest and highest genome indices"""
    import skani_b200 as sk
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
    genomes = small[:12] + empty + fam + empty + small[12:]
    s = sk.sketch_sequences(ctx, genomes)
    cards = [s.info(g)["n_markers"] for g in range(len(s))]
    assert min(cards) == 0 and any(0 < c < 20 for c in cards[:12]) and any(0 < c < 20 for c in cards[-12:])
    return s


@pytest.mark.parametrize("rescue", [True, False])
def test_small_and_empty_genomes(ctx, rescue):
    import skani_b200 as sk
    s = small_and_empty_set(ctx)
    n = len(s)
    rng = np.random.default_rng(3)
    lr = length_rank(s)
    for rank in (lr, (n - 1 - lr).astype(np.uint32), rng.permutation(n).astype(np.uint32)):   # small genomes last, first, anywhere
        for t in (0.8, 0.95):
            check(ctx, s, rank, t, sk.map_params(rescue_small=rescue))


def test_af_filters_make_sentinels(ctx):
    import skani_b200 as sk
    s = small_and_empty_set(ctx)
    for mp in (sk.map_params(min_af=0.5), sk.map_params(both_min_af=0.5)):
        tri = triangle_rows(ctx, s, mp)
        assert (tri["ani"] == -1).any()
        check(ctx, s, length_rank(s), 0.95, mp)


def test_empty_and_single(ctx):
    import skani_b200 as sk
    s = sk.sketch_sequences(ctx, [[b"ACGT" * 5000]])
    rep, cl, join, st = sk.dereplicate(ctx, s, np.zeros(1, np.uint32))
    assert rep.tolist() == [0] and cl.tolist() == [0] and np.isnan(join["ani"][0]) and st.n_clusters == 1 and st.pairs_chained == 0


def test_refusals(ctx):
    import ctypes as C
    import skani_b200 as sk
    from skani_b200 import _lib
    s, *_ = family_set(ctx, 6, 60_000, 3)
    for rank, msg in ((np.array([0, 0, 1, 2, 3, 4], np.uint32), "permutation"), (np.array([0, 1, 2, 3, 4, 6], np.uint32), "permutation")):
        with pytest.raises(sk.host.SkaniError, match=msg):
            sk.dereplicate(ctx, s, rank)
    with pytest.raises(sk.host.SkaniError, match="NaN"):
        sk.dereplicate(ctx, s, np.arange(6, dtype=np.uint32), min_ani=float("nan"))
    mp, dp, st = sk.map_params(), _lib.DerepParams(0.95, 0), _lib.DerepStats()
    rank = np.arange(6, dtype=np.uint32)
    o32 = np.zeros(6, np.uint32); join = np.zeros(6, sk.host.RESULT_DTYPE)
    args = [ctx.h, s.h, C.byref(mp), rank.ctypes.data, C.byref(dp), o32.ctypes.data, o32.ctypes.data, join.ctypes.data, C.byref(st)]
    for i in (1, 2, 3, 4, 5, 6, 7):
        bad = list(args)
        bad[i] = None
        assert ctx.L.sk_dereplicate(*bad) == -2
        assert "NULL" in ctx.L.sk_last_error(ctx.h).decode()
    assert ctx.L.sk_dereplicate(*args[:8], None) == 0     # stats may be NULL
    check(ctx, s, rank, 0.95, mp)                         # the context still works after every refusal
