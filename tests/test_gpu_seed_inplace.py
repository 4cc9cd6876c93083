"""GPU: a sketch set seeded in many sub-batches equals the same set seeded in one, array by array, and both equal seed_ref.

The records (pv_kmer / pv_pos / pv_cc) and each genome's raw markers come out of expand_kernel, which numbers a warp's
records by a scan of its units' pass masks and hands out marker slots per genome through counters; sub-batch edges, empty
genomes, genomes too short for a window, 'N'-rich contigs and dense sampling (c = 1: up to 32 records per unit) are where
that numbering can slip.  SK_SUBBATCH_BYTES=1 makes every genome boundary a sub-batch boundary.  Every array of the set
(position view, pv_mult, k-mer view, ukmer / ustart, markers, contig offsets and lengths, seed / group / marker / contig
offsets) is compared bit for bit; the k-mer tables are checked against ktable_ref's contract, genome by genome, in both
sets, including a genome of >= 2^20 records that takes the bucket-index fallback."""
import numpy as np
import pytest

import ktable_ref as T
import seed_cases as SC
import seed_ref as R
import test_gpu_seed_edges as E

pytestmark = pytest.mark.gpu

OFFSETS = ("seed_off", "uk_off", "mk_off", "ctg_off")


@pytest.fixture(scope="module")
def ctx():
    import skani_b200 as sk
    c = sk.Context(0)
    yield c
    c.close()


def n_rich(rng, n):
    s = SC.rand_acgt(rng, n)
    for p in rng.integers(0, n, n // 60):
        s[p:p + int(rng.integers(1, 30))] = ord("N")
    return s


def mixed_genomes(seed=31):
    """Random genomes with empty genomes, sub-window contigs (< 42 bases) and 'N'-rich contigs at genome (= sub-batch) edges"""
    rng = np.random.default_rng(seed)
    g = []
    for i in range(14):
        kind = i % 7
        if kind == 0:
            g.append([])                                                            # no contig at all
        elif kind == 1:
            g.append([SC.rand_acgt(rng, int(n)) for n in rng.integers(0, 42, 5)])    # no window at all
        elif kind == 2:
            g.append([n_rich(rng, int(rng.integers(2000, 9000))) for _ in range(3)])
        elif kind == 3:
            g.append([SC.rand_acgt(rng, int(n)) for n in rng.integers(1, 300, 40)])  # many contigs per unit range
        else:
            g.append([SC.rand_acgt(rng, int(rng.integers(5000, 40000))) for _ in range(int(rng.integers(1, 4)))])
    g[5] = g[5] + [SC.rand_acgt(rng, 30)]                                          # a short contig closing a genome
    return g


def one_and_many(ctx, monkeypatch, genomes, c, k, mc, avx2, path):
    one = E.sketch(ctx, genomes, c, k, mc, avx2, path, monkeypatch)
    monkeypatch.setenv("SK_SUBBATCH_BYTES", "1")
    try:
        many = E.sketch(ctx, genomes, c, k, mc, avx2, path, monkeypatch)
    finally:
        monkeypatch.delenv("SK_SUBBATCH_BYTES")
    return one, many


def check_tables(s, refs, m, a):
    """every genome's k-mer table follows the contract; returns the genomes without a table"""
    none = []
    for g, r in enumerate(refs):
        ht = a["htab"][m["ht_off"][g]:m["ht_off"][g + 1]]
        cnt = np.diff(r["ustart"]).astype(np.int64)
        if T.capacity(len(r["ukmer"]), len(r["pv_kmer"])) == 0:
            assert len(ht) == 0, g
            none.append(g)
        else:
            T.check_table(ht, r["ukmer"], r["ustart"][:-1], cnt)
    return none


def assert_same(one, many, genomes, c, k, mc, avx2):
    refs, m1, a1 = E.check_set(one, genomes, c, k, mc, avx2, export=False)
    _, m2, a2 = E.check_set(many, genomes, c, k, mc, avx2, refs=refs, export=False)
    for x in OFFSETS:
        assert np.array_equal(m1[x], m2[x]), x
    for x in E.ARRAYS[:-1]:
        assert np.array_equal(a1[x], a2[x]), x
    for s in (one, many):
        t = E.blob(s, E.TABLES)
        check_tables(s, refs, *t)
    for g in range(len(genomes)):
        e1, e2 = one.export(g), many.export(g)
        for key in ("kmer", "pos", "cc", "markers", "contig_lengths"):
            assert np.array_equal(e1[key], e2[key]), (g, key)
    return refs


@pytest.mark.parametrize("path", ["dev1", "host_pack0"])
@pytest.mark.parametrize("avx2", E.SEM, ids=E.SEM_IDS)
@pytest.mark.parametrize("c,mc", [(1, 1), (30, 60), (125, 1000)])
def test_sub_batches_equal_one_batch(ctx, monkeypatch, c, mc, avx2, path):
    genomes = mixed_genomes()
    one, many = one_and_many(ctx, monkeypatch, genomes, c, 15, mc, avx2, path)
    refs = assert_same(one, many, genomes, c, 15, mc, avx2)
    assert any(len(g) == 0 for g in genomes) and any(len(r["pv_kmer"]) == 0 and len(g) > 0 for g, r in zip(genomes, refs))
    assert sum(len(r["markers"]) for r in refs) > 0
    one.free(); many.free()


def test_bucket_fallback_genome_between_sub_batches(ctx, monkeypatch):
    rng = np.random.default_rng(32)
    big = [SC.rand_acgt(rng, (1 << 20) + 64)]                                  # c = 1: >= 2^20 records, no table
    genomes = [[SC.rand_acgt(rng, 3000)], big, [], [SC.rand_acgt(rng, 5000), SC.rand_acgt(rng, 40)]]
    one, many = one_and_many(ctx, monkeypatch, genomes, 1, 15, 50, True, "dev0")
    refs = assert_same(one, many, genomes, 1, 15, 50, True)
    assert len(refs[1]["pv_kmer"]) >= 1 << 20
    assert check_tables(many, refs, *E.blob(many, E.TABLES)) == [1, 2]
    one.free(); many.free()


@pytest.mark.parametrize("c,mc", [(1, 1), (125, 1000)])
def test_marker_multiset_per_genome(ctx, monkeypatch, c, mc):
    """the raw markers a genome collects (through the per-genome counters) dedup to the reference's marker set: checked on
    genomes whose contigs repeat, so the same marker arrives from several warps"""
    rng = np.random.default_rng(33)
    unit = SC.rand_acgt(rng, 7000)
    genomes = [[unit, unit.copy(), SC.rand_acgt(rng, 900)], [], [unit[::-1].copy()] * 3, [SC.rand_acgt(rng, 20000)]]
    s = E.sketch(ctx, genomes, c, 15, mc, True, "dev0", monkeypatch)
    for g, contigs in enumerate(genomes):
        want = np.unique(np.concatenate([R.contig_seeds(x, 15, c, mc)[3] for x in contigs] + [np.zeros(0, np.uint64)]))
        assert np.array_equal(s.export(g)["markers"], want.astype(np.uint64)), g
    s.free()
