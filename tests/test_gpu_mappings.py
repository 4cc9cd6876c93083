"""sk_chain_pairs_mappings / sk_chain_pairs_multi_mappings on the GPU against the CPU oracle: every pair's records equal the
restatement of mapping_ref.py (the oracle's kept intervals in the caller's orientation, joined to chunk_estimate of their
chunk, sorted), every integer field exactly and chunk_est within EST_ULPS (the device's pow() against glibc's, as in
test_gpu_chunkstat.py); and out equals sk_chain_pairs' byte for byte."""
import os

import numpy as np
import pytest

import oracle_py as O
import mapping_ref
from chain_testlib import EST_ULPS, make_sets, mutate, rand_seq, revcomp, synth_genomes, ulp_diff
from fasta_py import read_fastx

pytestmark = pytest.mark.gpu
GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
INT_FIELDS = ("query_contig", "ref_contig", "q0", "q1", "r0", "r1", "num_anchors", "chunk", "chunk_weight", "reverse", "switched",
              "chunk_valid", "pad")


@pytest.fixture(scope="module")
def ctx():
    import skani_b200 as sk
    c = sk.Context(0)
    yield c
    c.close()


def load_genome(name):
    return [np.frombuffer(s, np.uint8) for _, s in read_fastx(os.path.join(GOLD, name))]


def assert_records_equal(got, exp, what):
    assert len(got) == len(exp), (what, len(got), len(exp))
    for f in INT_FIELDS:
        bad = np.nonzero(got[f] != exp[f])[0]
        assert len(bad) == 0, (what, f, int(bad[0]), got[int(bad[0])], exp[int(bad[0])])
    assert int(ulp_diff(got["chunk_est"], exp["chunk_est"]).max(initial=0)) <= EST_ULPS, what


def run_and_check(ctx, gs, osk, pairs, mp, cp, c, k=15):
    """chains pairs both ways, checks out and every pair's records; returns (results, offsets, mappings)"""
    import skani_b200 as sk
    pairs = np.asarray(pairs, np.uint64)
    res, off, maps = sk.chain_pairs_mappings(ctx, gs, gs, pairs, mp)
    plain = sk.chain_pairs(ctx, gs, gs, pairs, mp, as_array=True)
    assert res.tobytes() == plain.tobytes()
    assert off[0] == 0 and np.all(np.diff(off.astype(np.int64)) >= 0) and off[-1] == len(maps)
    cache = {}
    for i, p in enumerate(pairs.tolist()):
        r, q = p >> 32, p & 0xFFFFFFFF
        if (r, q) not in cache:
            cache[(r, q)] = mapping_ref.expected(O.chain_debug(osk[r], osk[q], cp), c, k)
        assert_records_equal(maps[int(off[i]):int(off[i + 1])], cache[(r, q)], (i, r, q))
    return res, off, maps


def test_struct_layout():
    import ctypes as C
    import skani_b200 as sk
    dt = sk.MAPPING_DTYPE
    assert dt.itemsize == 48
    offs = {n: dt.fields[n][1] for n in dt.names}
    assert offs == dict(query_contig=0, ref_contig=4, q0=8, q1=12, r0=16, r1=20, num_anchors=24, chunk=28, chunk_est=32,
                        chunk_weight=40, reverse=44, switched=45, chunk_valid=46, pad=47)
    assert C.sizeof(C.c_double) == 8


@pytest.mark.parametrize("c", [125, 200])
def test_ecoli_both_orientations(ctx, c):
    import skani_b200 as sk
    kw = dict(c=c, k=15, marker_c=1000)
    gs, osk = make_sets(ctx, [load_genome("e.coli-EC590.fasta.gz"), load_genome("e.coli-K12.fasta.gz")], kw)
    res, off, maps = run_and_check(ctx, gs, osk, [(0 << 32) | 1, (1 << 32) | 0], sk.map_params(), O.cmd(), c)
    sw = [set(maps[int(off[i]):int(off[i + 1])]["switched"].tolist()) for i in range(2)]
    assert sorted(map(tuple, sw)) == [(0,), (1,)], sw          # one orientation is switched, the other not
    assert all(off[i + 1] - off[i] > 100 for i in range(2))
    # switch_qr picks the same roles both ways, so the records of (a, b) are those of (b, a) with the sides swapped
    a, b = maps[int(off[0]):int(off[1])], maps[int(off[1]):int(off[2])]
    fa = {(int(m["query_contig"]), int(m["q0"]), int(m["q1"]), int(m["ref_contig"]), int(m["r0"]), int(m["r1"]), int(m["reverse"]),
           int(m["chunk"])) for m in a}
    fb = {(int(m["ref_contig"]), int(m["r0"]), int(m["r1"]), int(m["query_contig"]), int(m["q0"]), int(m["q1"]), int(m["reverse"]),
           int(m["chunk"])) for m in b}
    assert fa == fb and len(fa) == len(a)


@pytest.mark.parametrize("kw", [dict(robust=True), dict(median=True), dict(learned_ani=False)])
def test_trim_modes(ctx, kw):
    import skani_b200 as sk
    gs, osk = make_sets(ctx, [load_genome("e.coli-EC590.fasta.gz"), load_genome("e.coli-K12.fasta.gz")], dict(c=125, k=15, marker_c=1000))
    run_and_check(ctx, gs, osk, [(0 << 32) | 1, (1 << 32) | 0], sk.map_params(**kw), O.cmd(**kw), 125)


def test_viruses_individual(ctx):
    import skani_b200 as sk
    ctgs = [np.frombuffer(s, np.uint8) for _, s in read_fastx(os.path.join(GOLD, "viruses.fna"))]
    kw = dict(c=125, k=15, marker_c=1000)
    gs, osk = make_sets(ctx, [ctgs], kw, individual=True)
    n = len(osk)
    pairs = [(i << 32) | j for i in range(n) for j in range(n) if i != j]
    run_and_check(ctx, gs, osk, pairs, sk.map_params(learned_ani=False), O.cmd(learned_ani=False), 125)


def planted_pair(seed=5, L=300_000, seg=60_000, rate=0.02):
    """a reference and a query that carries a mutated copy of ref[50k:50k+seg] forward and one of ref[200k:200k+seg] reverse-
    complemented, in an unrelated background"""
    rng = np.random.default_rng(seed)
    ref = rand_seq(rng, L)
    q = rand_seq(rng, L)
    q[20_000:20_000 + seg] = mutate(rng, ref[50_000:50_000 + seg], rate)
    q[150_000:150_000 + seg] = mutate(rng, revcomp(ref[200_000:200_000 + seg]), rate)
    return ref, q


def test_reverse_strand_and_result_kinds(ctx):
    """- strand records; pairs ending in a valid ANI, in -1 (AF cutoff) and in NaN (no anchors / no estimate)"""
    import skani_b200 as sk
    rng = np.random.default_rng(11)
    ref, q = planted_pair()
    small = mutate(rng, ref[100_000:103_000], 0.01)          # 3 kb shared by a 300 kb genome: AF far below 15 %
    unrelated = rand_seq(rng, 300_000)
    short = mutate(rng, ref[120_000:120_400], 0.0)           # < MIN_LENGTH_COVER of shared sequence
    genomes = [[ref], [q], [np.concatenate([small, rand_seq(rng, 297_000)])], [unrelated],
               [np.concatenate([rand_seq(rng, 50_000), short, rand_seq(rng, 50_000)])]]
    kw = dict(c=125, k=15, marker_c=1000)
    gs, osk = make_sets(ctx, genomes, kw)
    mp, cp = sk.map_params(learned_ani=False), O.cmd(learned_ani=False)
    pairs = [(0 << 32) | j for j in range(1, 5)] + [(j << 32) | 0 for j in range(1, 5)]
    res, off, maps = run_and_check(ctx, gs, osk, pairs, mp, cp, 125)
    assert set(maps[int(off[0]):int(off[1])]["reverse"].tolist()) == {0, 1}
    kinds = set()
    for i, r in enumerate(res):
        kinds.add("nan" if np.isnan(r["ani"]) else "-1" if r["ani"] == -1 else "ani")
        if np.isnan(r["ani"]) and off[i + 1] > off[i]:
            kinds.add("nan with intervals")
    assert {"nan", "-1", "ani"} <= kinds, kinds


def test_weighted_mean_invariant(ctx):
    """--no-learned-ani, no trimming: sum(w * est) / sum(w) over the pair's distinct valid chunks is the ANI (f32)"""
    import skani_b200 as sk
    gs, osk = make_sets(ctx, [load_genome("e.coli-EC590.fasta.gz"), load_genome("e.coli-K12.fasta.gz")], dict(c=125, k=15, marker_c=1000))
    res, off, maps = sk.chain_pairs_mappings(ctx, gs, gs, np.array([(0 << 32) | 1, (1 << 32) | 0], np.uint64), sk.map_params(learned_ani=False))
    for i in range(2):
        m = maps[int(off[i]):int(off[i + 1])]
        ch = {}
        for x in m[m["chunk_valid"] != 0]:
            ch[int(x["chunk"])] = (float(x["chunk_est"]), int(x["chunk_weight"]))
        est = np.array([e for e, _ in ch.values()]); w = np.array([w for _, w in ch.values()], np.float64)
        assert abs(np.float32((est * w).sum() / w.sum()) - res[i]["ani"]) <= 2 * np.spacing(np.float32(res[i]["ani"]))


def test_many_batches(ctx):
    """more than one chain batch (65 535 pairs each): records land with their pairs across batch boundaries"""
    import skani_b200 as sk
    genomes = synth_genomes(6, 60_000, 3)
    gs, osk = make_sets(ctx, genomes, dict(c=125, k=15, marker_c=1000))
    base = [(i << 32) | j for i in range(6) for j in range(6) if i != j]
    pairs = np.array((base * (140_000 // len(base) + 1))[:140_000], np.uint64)
    res, off, maps = sk.chain_pairs_mappings(ctx, gs, gs, pairs, sk.map_params())
    assert res.tobytes() == sk.chain_pairs(ctx, gs, gs, pairs, sk.map_params(), as_array=True).tobytes()
    first = {}
    for i, p in enumerate(pairs.tolist()):
        m = maps[int(off[i]):int(off[i + 1])].tobytes()
        if p not in first:
            first[p] = m
            exp = mapping_ref.expected(O.chain_debug(osk[p >> 32], osk[p & 0xFFFFFFFF], O.cmd()), 125, 15)
            assert_records_equal(maps[int(off[i]):int(off[i + 1])], exp, p)
        else:
            assert m == first[p], (i, p)
    assert sum(off[i + 1] > off[i] for i in range(len(base))) > 0


def test_multi_two_contexts_equal_one(ctx):
    """refs split into two blocks on two contexts of one device give the records of the one-context call, in pair order"""
    import skani_b200 as sk
    genomes = [load_genome("e.coli-EC590.fasta.gz"), load_genome("e.coli-K12.fasta.gz")] + synth_genomes(4, 200_000, 2)
    n = len(genomes)
    pairs = np.array([(i << 32) | j for i in range(n) for j in range(n) if i != j][::-1], np.uint64)
    mp = sk.map_params()
    sp = sk.sketch_params(c=125, k=15, marker_c=1000)
    rall = sk.sketch_sequences(ctx, genomes, sp)
    q0 = sk.sketch_sequences(ctx, genomes, sp)
    one = sk.chain_pairs_multi_mappings([ctx], [rall], [0], [q0], pairs, mp)
    assert one[1][-1] > 0
    ctx2 = sk.Context(0)
    try:
        r0 = sk.sketch_sequences(ctx, genomes[:3], sp)
        r1 = sk.sketch_sequences(ctx2, genomes[3:], sp)
        q1 = q0.copy_to(ctx2)
        two = sk.chain_pairs_multi_mappings([ctx, ctx2], [r0, r1], [0, 3], [q0, q1], pairs, mp)
        plain = sk.chain_pairs_multi([ctx, ctx2], [r0, r1], [0, 3], [q0, q1], pairs, mp, as_array=True)
        assert two[0].tobytes() == plain.tobytes() == one[0].tobytes()
        assert np.array_equal(two[1], one[1])
        assert two[2].tobytes() == one[2].tobytes()
        for s in (r1, q1):
            s.free()
    finally:
        ctx2.close()
