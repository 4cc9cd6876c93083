"""sk_dereplicate_fixed (skani_b200.dereplicate_fixed) against sk_cluster's greedy clusters of the same set's triangle rows
(screen_triangle + chain_pairs) without the rows between two fixed genomes: rep and cluster equal, every member's join byte
for byte the row sk_cluster's edge points to, and pairs_screened, pairs_chained and waves equal to tests/derep_fixed_ref.py's
counts on the triangle's pairs.  n_fixed = 0 is sk_dereplicate byte for byte, stats counts and kernel launches included.
Synthetic families with contiguous and shuffled ids; fixed sets of no genome, one, a few, half, all but one and all; fixed
sets holding whole families (edges inside the fixed set); the representatives of an earlier run over part of the genomes
(then also equal to plain sk_dereplicate); wave sizes 1, 3 and the default; the E. coli goldens; viruses per record (-i);
genomes under 20 markers and without markers, fixed at low or high genome indices, with the rescue on and off; refusals."""
import os

import numpy as np
import pytest

import derep_fixed_ref as F
from bench_support import synth
from fasta_py import read_fastx

pytestmark = pytest.mark.gpu

GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
WAVES = (1, 3, 0)
COUNTS = ("pairs_screened", "pairs_chained", "n_edges", "n_clusters", "waves", "rounds")


@pytest.fixture(scope="module")
def ctx():
    import skani_b200 as sk
    c = sk.Context(0)
    yield c
    c.close()


def length_rank(s):
    total = np.array([s.info(g)["total_len"] for g in range(len(s))], np.int64)
    order = np.lexsort((np.arange(len(s)), -total))
    rank = np.empty(len(s), np.uint32)
    rank[order] = np.arange(len(s))
    return rank


def fixed_first(first, n, then=None):
    """the rank that puts the genomes of `first` first in that order, then the others in the order of `then` (ascending index)"""
    first = [int(g) for g in first]
    taken = set(first)
    rest = [int(g) for g in (range(n) if then is None else np.argsort(then, kind="stable")) if int(g) not in taken]
    rank = np.empty(n, np.uint32)
    rank[np.array(first + rest, np.int64)] = np.arange(n, dtype=np.uint32)
    return rank


def triangle(ctx, s, mp):
    """the triangle's pair keys and their chained rows"""
    import skani_b200 as sk
    pairs = np.asarray(sk.screen_triangle(ctx, s, mp), np.uint64)
    return pairs, sk.chain_pairs(ctx, s, s, pairs, mp, as_array=True)


def check(ctx, s, rank, n_fixed, min_ani, mp, waves=WAVES, tri=None):
    """dereplicate_fixed at every wave size equals cluster (greedy) on the triangle's rows without F x F, with the restatement's
    counts; returns (rep, cluster, join, stats) of the last wave size and whether F holds an edge"""
    import skani_b200 as sk
    n = len(s)
    pairs, rows = tri if tri is not None else triangle(ctx, s, mp)
    fixed = np.zeros(n, bool)
    fixed[np.argsort(rank, kind="stable")[:n_fixed]] = True
    keep = ~(fixed[rows["ref_id"]] & fixed[rows["query_id"]])
    kept = rows[keep]
    erep, ecl, eedge, _ = sk.cluster(ctx, n, kept, rank, min_ani=min_ani)
    g = np.arange(n)
    mem = erep != g
    screen = {(int(p >> np.uint64(32)), int(p & np.uint64(0xFFFFFFFF))) for p in pairs}
    ani = {(int(p >> np.uint64(32)), int(p & np.uint64(0xFFFFFFFF))): np.float32(r) for p, r in zip(pairs, rows["ani"])}
    for w in waves:
        rep, cl, join, st = sk.dereplicate_fixed(ctx, s, rank, n_fixed, min_ani=min_ani, mp=mp, wave=w)
        assert np.array_equal(rep, erep) and np.array_equal(cl, ecl), (n_fixed, w, np.nonzero((rep != erep) | (cl != ecl))[0][:5])
        assert join[mem].tobytes() == kept[eedge[mem].astype(np.int64)].tobytes(), (n_fixed, w)
        assert np.isnan(join["ani"][~mem]).all()
        assert np.array_equal(join["ref_id"][~mem], g[~mem]) and np.array_equal(join["query_id"][~mem], g[~mem])
        assert (rep[fixed] == g[fixed]).all() and np.array_equal(np.sort(cl[fixed]), np.arange(n_fixed))
        _, _, _, chained, screened, nw = F.dereplicate(n, screen, ani, min_ani, rank, w, n_fixed)
        assert (st.pairs_screened, st.pairs_chained, st.waves) == (screened, len(chained), nw), (n_fixed, w)
        assert st.n_clusters == int((~mem).sum())
    with np.errstate(invalid="ignore"):
        inside = bool((~keep & (rows["ani"] > np.float32(0.1)) & (rows["ani"] >= np.float32(min_ani))).any())
    return (rep, cl, join, st), inside


def fixed_sizes(n):
    return sorted({0, 1, 3, n // 2, n - 1, n})


def family_set(ctx, n, L, G, shuffled=False):
    import skani_b200 as sk
    bases, off, goc = synth.generate_ids(synth.shuffled_ids(n, 5), L, G=G) if shuffled else synth.generate(0, n, L, G=G)
    return sk.sketch_contigs(ctx, bases, off, goc, n), bases, off, goc


def test_no_fixed_is_dereplicate(ctx):
    """n_fixed = 0: sk_dereplicate's outputs byte for byte, its stats counts and as many kernel launches"""
    import skani_b200 as sk
    s, *_ = family_set(ctx, 120, 100_000, 20, shuffled=True)
    mp = sk.map_params()
    for rank in (length_rank(s), np.random.default_rng(2).permutation(len(s)).astype(np.uint32)):
        for w in WAVES:
            l0 = ctx.launches
            exp = sk.dereplicate(ctx, s, rank, min_ani=0.95, mp=mp, wave=w)
            l1 = ctx.launches
            got = sk.dereplicate_fixed(ctx, s, rank, 0, min_ani=0.95, mp=mp, wave=w)
            l2 = ctx.launches
            for a, b in zip(got[:3], exp[:3]):
                assert a.tobytes() == b.tobytes(), w
            for f in COUNTS:
                assert getattr(got[3], f) == getattr(exp[3], f), (w, f)
            assert l2 - l1 == l1 - l0 > 0, (w, l1 - l0, l2 - l1)


@pytest.mark.parametrize("shuffled", [False, True])
def test_synthetic_families(ctx, shuffled):
    import skani_b200 as sk
    s, *_ = family_set(ctx, 160, 100_000, 20, shuffled)
    mp = sk.map_params()
    tri = triangle(ctx, s, mp)
    rng = np.random.default_rng(3)
    for rank in (length_rank(s), rng.permutation(len(s)).astype(np.uint32)):
        for n_fixed in fixed_sizes(len(s)):
            for t in (0.95, 0.99):
                (rep, cl, join, st), _ = check(ctx, s, rank, n_fixed, t, mp, tri=tri)
                if n_fixed == len(s):
                    assert st.waves == 0 and st.pairs_screened == 0 and st.pairs_chained == 0


def test_fixed_families_keep_every_genome(ctx):
    """F = three whole families (contiguous ids, ranked first): edges inside F, and every fixed genome stays a representative"""
    import skani_b200 as sk
    s, *_ = family_set(ctx, 100, 100_000, 10)
    mp = sk.map_params()
    rank = np.arange(len(s), dtype=np.uint32)
    (rep, _, _, _), inside = check(ctx, s, rank, 30, 0.95, mp)
    assert inside
    prep = sk.dereplicate(ctx, s, rank, min_ani=0.95, mp=mp)[0]
    assert (rep[:30] == np.arange(30)).all() and not (prep[:30] == np.arange(30)).all()


@pytest.mark.parametrize("shuffled", [False, True])
def test_representatives_of_an_earlier_run(ctx, shuffled):
    """an earlier run over the first 100 of 160 genomes; its representatives fixed (in their old rank order) and the other
    genomes added: the result is plain sk_dereplicate's on the same ranks, and the representatives keep their cluster ids"""
    import skani_b200 as sk
    n, m = 160, 100
    s, bases, off, goc = family_set(ctx, n, 100_000, 20, shuffled)
    mp = sk.map_params()
    idx = np.nonzero(goc < m)[0]
    old = sk.sketch_contigs(ctx, bases[:int(off[idx[-1] + 1])], off[:idx[-1] + 2], goc[idx], m)
    orank = length_rank(old)
    orep, ocl, _, _ = sk.dereplicate(ctx, old, orank, min_ani=0.95, mp=mp)
    reps = [g for g in np.argsort(orank, kind="stable") if orep[g] == g]
    rank = fixed_first(reps, n, length_rank(s))
    (rep, cl, join, st), inside = check(ctx, s, rank, len(reps), 0.95, mp)
    assert not inside
    prep, pcl, pjoin, pst = sk.dereplicate(ctx, s, rank, min_ani=0.95, mp=mp)
    assert np.array_equal(rep, prep) and np.array_equal(cl, pcl) and join.tobytes() == pjoin.tobytes()
    assert np.array_equal(cl[reps], ocl[reps])
    print("adding %d genomes to %d representatives: %d pairs screened, %d chained; a full run: %d, %d"
          % (n - m, len(reps), st.pairs_screened, st.pairs_chained, pst.pairs_screened, pst.pairs_chained))


def _ecoli():
    return [[seq for _, seq in read_fastx(os.path.join(GOLD, f))] for f in ("e.coli-EC590.fasta.gz", "e.coli-K12.fasta.gz")]


def test_ecoli_goldens(ctx):
    import skani_b200 as sk
    s = sk.sketch_sequences(ctx, _ecoli())
    mp = sk.map_params()
    tri = triangle(ctx, s, mp)
    for rank in ([0, 1], [1, 0]):
        for n_fixed in (0, 1, 2):
            for t in (0.95, 0.99, 0.999):
                check(ctx, s, np.array(rank, np.uint32), n_fixed, t, mp, tri=tri)


def test_viruses_individual(ctx):
    import skani_b200 as sk
    recs = [seq for _, seq in read_fastx(os.path.join(GOLD, "viruses.fna"))]
    s = sk.sketch_sequences(ctx, [recs], individual_contig=True)
    n = len(s)
    mp = sk.map_params(learned_ani=False)
    tri = triangle(ctx, s, mp)
    for n_fixed in fixed_sizes(n):
        for t in (0.8, 0.95):
            check(ctx, s, length_rank(s), n_fixed, t, mp, tri=tri)


def small_and_empty_set(ctx):
    """families of 100 kbp genomes between 12 slices of family members of 3-25 kbp (about 3-25 markers) and a poly-A genome
    without markers at each end of the genome indices"""
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
    s = sk.sketch_sequences(ctx, small[:12] + empty + fam + empty + small[12:])
    cards = [s.info(g)["n_markers"] for g in range(len(s))]
    assert min(cards) == 0 and any(0 < c < 20 for c in cards[:12]) and any(0 < c < 20 for c in cards[-12:])
    return s


@pytest.mark.parametrize("rescue", [True, False])
def test_small_and_empty_genomes(ctx, rescue):
    """fixed: the small and empty genomes at low indices (the fixed genome is the smaller index of its pairs), those at high
    indices (the larger), or family genomes between them"""
    import skani_b200 as sk
    s = small_and_empty_set(ctx)
    n = len(s)
    mp = sk.map_params(rescue_small=rescue)
    tri = triangle(ctx, s, mp)
    lr = length_rank(s)
    for first in (range(13), range(n - 13, n), range(13, 43)):
        rank = fixed_first(first, n, lr)
        for n_fixed in (1, 5, len(first)):
            for t in (0.8, 0.95):
                check(ctx, s, rank, n_fixed, t, mp, tri=tri)


def test_refusals(ctx):
    import ctypes as C
    import skani_b200 as sk
    from skani_b200 import _lib
    s, *_ = family_set(ctx, 6, 60_000, 3)
    rank = np.arange(6, dtype=np.uint32)
    with pytest.raises(sk.host.SkaniError, match="fixed representatives, more than the 6 genomes"):
        sk.dereplicate_fixed(ctx, s, rank, 7)
    with pytest.raises(sk.host.SkaniError, match="permutation"):
        sk.dereplicate_fixed(ctx, s, np.array([0, 0, 1, 2, 3, 4], np.uint32), 2)
    with pytest.raises(sk.host.SkaniError, match="NaN"):
        sk.dereplicate_fixed(ctx, s, rank, 2, min_ani=float("nan"))
    mp, dp, st = sk.map_params(), _lib.DerepParams(0.95, 0), _lib.DerepStats()
    o32 = np.zeros(6, np.uint32); join = np.zeros(6, sk.host.RESULT_DTYPE)
    args = [ctx.h, s.h, C.byref(mp), rank.ctypes.data, 2, C.byref(dp), o32.ctypes.data, o32.ctypes.data, join.ctypes.data, C.byref(st)]
    for i in (1, 2, 3, 5, 6, 7, 8):
        bad = list(args)
        bad[i] = None
        assert ctx.L.sk_dereplicate_fixed(*bad) == -2
        assert "sk_dereplicate_fixed: NULL" in ctx.L.sk_last_error(ctx.h).decode()
    assert ctx.L.sk_dereplicate_fixed(*args[:9], None) == 0     # stats may be NULL
    check(ctx, s, rank, 6, 0.95, mp)                             # the context still works after every refusal
