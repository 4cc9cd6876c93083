"""GPU parity of whole chaining batches against the CPU oracle, per pair and bit-exact, through sk_chain_pairs_debug (the
batching, descriptors and kernel instantiations of sk_chain_pairs, plus the per-anchor DP taps).  Each test asserts that
its input reached the edge it is named for: odd record offsets inside a batch, tiles of more than 1,024 anchors, records
whose anchors straddle an emission round, exact multiplicity limits, tile-aligned record counts, anchor-free tiles, the
chunk-staging bound, every DP variant, the 2^20-record probe threshold and more than one batch of pairs.

One comparison is narrower than assert_debug_equal on purpose: the reference reports switched = true for every pair
without anchors (src/chain.rs:714-720) whatever roles it chose, so for those pairs only the anchor-free outcome is compared
(assert_pair_equal).  Pairs with anchors are compared in full."""
import numpy as np
import pytest

import oracle_py as O
from chain_testlib import (TOL, assert_debug_equal, assert_result_close, make_sets, mutate, rand_seq, revcomp,
                           synth_genomes)

pytestmark = pytest.mark.gpu
TILE = 1024                     # query-role records per chunk_anchor_kernel tile, anchors per emission round
MAX_PAIRS_PER_BATCH = 65535


@pytest.fixture(scope="module")
def ctx():
    import skani_b200 as sk
    c = sk.Context(0)
    yield c
    c.close()


def pair_ids(pairs):
    return np.array([(r << 32) | q for r, q in pairs], np.uint64)


def roles(gd, r, q):
    """(query-role genome, ref-role genome) of the pair: the query role is iterated and chunked, the ref role probed."""
    return (r, q) if gd["switched"] else (q, r)


def assert_pair_equal(gd, od):
    """assert_debug_equal; the reference reports switched = true for every pair without anchors (src/chain.rs:714-720),
    whatever roles it chose, so there only the anchor-free outcome is compared"""
    if len(od["anchors"]) == 0:
        assert od["switched"] and len(gd["anchors"]) == 0
        gd = dict(gd, switched=True)
    assert_debug_equal(gd, od)


def check_batch(ctx, gs, osk, pairs, mp=None, cp=None):
    """sk_chain_pairs_debug over the whole list: every pair bit-exact against the oracle, and its results byte-identical to
    sk_chain_pairs on the same list.  Returns the debug dicts."""
    import skani_b200 as sk
    mp = mp or sk.map_params()
    cp = cp or O.cmd()
    gds = sk.chain_pairs_debug(ctx, gs, gs, pair_ids(pairs), mp)
    res = sk.chain_pairs(ctx, gs, gs, pair_ids(pairs), mp, as_array=True)
    got = np.frombuffer(b"".join(bytes(gd["result"]) for gd in gds), res.dtype)
    assert got.tobytes() == res.tobytes()
    for (r, q), gd in zip(pairs, gds):
        try:
            assert_pair_equal(gd, O.chain_debug(osk[r], osk[q], cp))
        except AssertionError as e:
            raise AssertionError("pair (%d, %d): %s" % (r, q, e)) from e
    return gds


def record_index(exp, anchors):
    """record index (in the query-role genome's (contig, pos) order) of every anchor"""
    key = np.sort(((exp["cc"].astype(np.uint64) >> np.uint64(1)) << np.uint64(32)) | exp["pos"].astype(np.uint64))
    assert np.all(np.diff(key.astype(np.int64)) > 0)           # one record per (contig, position)
    akey = (anchors[:, 0].astype(np.uint64) << np.uint64(32)) | anchors[:, 1].astype(np.uint64)
    idx = np.searchsorted(key, akey)
    assert np.array_equal(key[idx], akey)
    return idx


def tile_stats(exp, anchors):
    """(anchors per tile, number of records whose anchors straddle an emission round, largest anchor count of a record)"""
    n_rec = len(exp["pos"])
    n_tiles = (n_rec + TILE - 1) // TILE
    if len(anchors) == 0:
        return np.zeros(n_tiles, np.int64), 0, 0
    ri = record_index(exp, anchors)
    per_tile = np.bincount(ri // TILE, minlength=n_tiles)
    tile_first = np.concatenate([[0], np.cumsum(per_tile)])[ri // TILE]
    rnd = (np.arange(len(ri)) - tile_first) // TILE              # emission round of every anchor inside its tile
    starts = np.concatenate([[True], ri[1:] != ri[:-1]])
    ends = np.concatenate([ri[1:] != ri[:-1], [True]])
    straddle = int(np.sum(rnd[starts] != rnd[ends]))
    return per_tile, straddle, int(np.bincount(ri).max())


# ---------------------------------------------------------------------------------------------------------------------
# 1. a mixed batch: odd record offsets, empty and invalid pairs, self pairs, both roles, small and large ref-role tables
# ---------------------------------------------------------------------------------------------------------------------
EMPTY = 7          # genome slot without contigs: its pairs are invalid


def mixed_genomes():
    rng = np.random.default_rng(101)
    big = synth_genomes(6, 300_000, 3)                        # slots 0-2 and 3-5: two related clusters, multi-contig
    src = np.concatenate(big[0])
    g = [list(x) for x in big]
    g.append([src[1000:50_000].copy()])                       # slot 6: a 49 kb piece of slot 0 (one contig)
    g.append([])                                              # slot 7: no contigs
    for i in range(8):                                        # slots 8-15: small genomes (<= 1024 distinct k-mers), related
        a = 5_000 * i
        L = 9_000 + 1_371 * i
        g.append([mutate(rng, src[a:a + L], 0.01)])
    g.append([rand_seq(rng, 40_000)])                         # slot 16: unrelated to everything
    return g


def mixed_sets(ctx, genomes, kw):
    import skani_b200 as sk
    contigs, goc = [], []
    for gi, cs in enumerate(genomes):
        for c in cs:
            contigs.append(np.asarray(c, np.uint8)); goc.append(gi)
    bases = np.concatenate(contigs)
    off = np.concatenate([[0], np.cumsum([len(c) for c in contigs])]).astype(np.uint64)
    gs = sk.sketch_contigs(ctx, bases, off, np.asarray(goc, np.uint32), len(genomes), sk.sketch_params(**kw))
    osk = [O.sketch_from_contigs("g%06d" % gi, cs, **kw) if cs else None for gi, cs in enumerate(genomes)]
    return gs, osk


SMALL = list(range(8, 16))
MAJORITY_SMALL = ([(a, b) for a in SMALL[:5] for b in SMALL[:5] if a != b] + [(0, 8), (9, 1), (6, 10), (11, 6)] +
                  [(0, 1), (2, 0), (3, 3), (0, EMPTY), (EMPTY, 12), (16, 9), (13, 16), (4, 5), (12, 12), (15, 14)])
MINORITY_SMALL = ([(0, 1), (1, 0), (0, 2), (2, 1), (3, 4), (5, 3), (4, 5), (0, 0), (5, 5), (0, 3), (4, 1), (6, 0), (1, 6),
                   (0, EMPTY), (EMPTY, 3), (16, 0), (2, 16), (6, 2), (3, 6)] +
                  [(8, 0), (1, 9), (10, 11), (12, 13), (14, 6), (15, 8), (9, 9), (0, 15)])


def small_table(gs, g):
    """ref-role hash table of at most 2,048 entries (<= 1,024 distinct k-mers): staged in shared memory by the probe"""
    nk = gs.info(g)["n_kmers"]
    return 0 < nk <= 1024


@pytest.mark.parametrize("env", [{}, {"SK_PROBE_TMA": "0"}, {"SK_FORCE_BUCKET_PROBE": "1"}, {"SK_DP_GL": "8"}],
                         ids=["default", "no_tma", "bucket_probe", "dp_gl8"])
@pytest.mark.parametrize("mix", ["majority_small", "minority_small"])
def test_mixed_batch_every_pair_bit_exact(ctx, monkeypatch, env, mix):
    for k, v in env.items():
        monkeypatch.setenv(k, v)
    kw = dict(c=125, k=15, marker_c=1000)
    gs, osk = mixed_sets(ctx, mixed_genomes(), kw)
    assert gs.info(EMPTY)["n_contigs"] == 0
    pairs = MAJORITY_SMALL if mix == "majority_small" else MINORITY_SMALL
    import skani_b200 as sk
    gds = sk.chain_pairs_debug(ctx, gs, gs, pair_ids(pairs), sk.map_params())
    res = sk.chain_pairs(ctx, gs, gs, pair_ids(pairs), sk.map_params(), as_array=True)
    assert np.frombuffer(b"".join(bytes(gd["result"]) for gd in gds), res.dtype).tobytes() == res.tobytes()
    rec_off, odd_n, even_n, odd_off_hit, n_small, n_valid_empty = 0, 0, 0, 0, 0, 0
    for (r, q), gd in zip(pairs, gds):
        if EMPTY in (r, q):                                   # invalid pair: nothing is chained, no estimate
            assert len(gd["anchors"]) == 0 and len(gd["chunk_first"]) == 1 and len(gd["intervals"]) == 0
            assert np.isnan(gd["result"].ani)
            continue
        assert_pair_equal(gd, O.chain_debug(osk[r], osk[q], O.cmd()))
        qr, rr = roles(gd, r, q)
        n = gs.info(qr)["n_records"]
        if len(gd["anchors"]):
            odd_off_hit += rec_off & 1
            odd_n += n & 1
            even_n += 1 - (n & 1)
        else:
            n_valid_empty += 1
        n_small += small_table(gs, rr)
        rec_off += n
    assert odd_off_hit >= 1, "no pair with anchors starts at an odd record offset (the rec_nh halfword realignment)"
    assert odd_n >= 2 and even_n >= 2
    assert n_valid_empty >= 2, "no valid pair without anchors"
    if "SK_FORCE_BUCKET_PROBE" not in env:
        if mix == "majority_small":
            assert 2 * n_small >= len(pairs) and n_small < len(pairs) - 2   # staged probe, some global-memory tables
        else:
            assert 2 * n_small < len(pairs) and n_small >= 5                 # unstaged probe with small tables


# ---------------------------------------------------------------------------------------------------------------------
# 2. repeat units: many anchors per record, multi-round tiles, multiplicity exactly band and band + 1 on both sides
# ---------------------------------------------------------------------------------------------------------------------
def repeat_pair(c, seed):
    """(ref-role genome, query-role genome) built from repeat units; every k-mer multiplicity edge is placed on purpose"""
    band = 2500 // c
    rng = np.random.default_rng(seed)
    unit = rand_seq(rng, 2_500)
    e_ref = [rand_seq(rng, 1_500) for _ in range(2)]       # occur band / band + 1 times in the ref role, once in the query role
    e_qry = [rand_seq(rng, 1_500) for _ in range(2)]       # occur band / band + 1 times in the query role, once in the ref role
    backbone = rand_seq(rng, 400_000)

    def spacer():
        return rand_seq(rng, 400)

    def copies(u, n):                                      # exact copies, every other one reverse-complemented
        out = []
        for i in range(n):
            out += [revcomp(u) if i & 1 else u, spacer()]
        return out

    n_ref_units, n_qry_units = min(band - 2, 40), 12
    ref = [backbone]
    for _ in range(n_ref_units):
        ref += [mutate(rng, unit, 0.01), spacer()]
    ref += copies(e_ref[0], band) + copies(e_ref[1], band + 1) + [e_qry[0], spacer(), e_qry[1]]
    qry = [mutate(rng, backbone[:150_000], 0.01)]
    for _ in range(n_qry_units):
        qry += [mutate(rng, unit, 0.01), spacer()]
    qry += [e_ref[0], spacer(), revcomp(e_ref[1]), spacer()] + copies(e_qry[0], band) + copies(e_qry[1], band + 1)
    qry += [mutate(rng, backbone[150_000:200_000], 0.01)]
    return np.concatenate(ref), np.concatenate(qry), band


def kmer_counts(exp):
    k, n = np.unique(exp["kmer"], return_counts=True)
    return dict(zip(k.tolist(), n.tolist()))


@pytest.mark.parametrize("c", [125, 30])
def test_repeat_units_multi_round_tiles_and_multiplicity_edges(ctx, c):
    ref, qry, band = repeat_pair(c, 5 + c)
    kw = dict(c=c, k=15, marker_c=1000 if c >= 100 else 200)
    gs, osk = make_sets(ctx, [[ref], [qry], [mutate(np.random.default_rng(3), qry, 0.005)]], kw)
    pairs = [(0, 1), (1, 0), (0, 2), (1, 2), (2, 1)]
    gds = check_batch(ctx, gs, osk, pairs)
    gd = gds[0]
    qr, rr = roles(gd, 0, 1)
    assert (qr, rr) == (1, 0), "the repeat-rich query genome must be the iterated one"
    eq, er = gs.export(qr), gs.export(rr)
    cq, cr = kmer_counts(eq), kmer_counts(er)
    # multiplicity edges reached on both sides by k-mers the other genome holds
    assert any(n == band and k in cq for k, n in cr.items()), "no ref-role k-mer with multiplicity == band hit"
    assert any(n == band + 1 and k in cq for k, n in cr.items()), "no ref-role k-mer with multiplicity == band + 1 hit"
    assert any(n == band and k in cr for k, n in cq.items()), "no query-role k-mer with multiplicity == band"
    assert any(n == band + 1 and k in cr for k, n in cq.items()), "no query-role k-mer with multiplicity == band + 1"
    per_tile, straddle, max_nh = tile_stats(eq, gd["anchors"])
    assert max_nh == band, (max_nh, band)                  # a record carries exactly band anchors, none carries more
    assert per_tile.max() > TILE, per_tile                 # a tile emits in several rounds
    assert straddle > 0                                    # some record's anchors are split between two rounds


# ---------------------------------------------------------------------------------------------------------------------
# 3 + 4. tile-aligned query-role genomes (record counts cut by bisection on the GPU sketcher) and the chunk-staging bound
# ---------------------------------------------------------------------------------------------------------------------
def n_records(ctx, contigs, kw):
    import skani_b200 as sk
    return sk.sketch_sequences(ctx, [contigs], sk.sketch_params(**kw)).info(0)["n_records"]


def cut_to_records(ctx, head, seq, target, kw):
    """shortest prefix of seq such that the genome head + [prefix] has exactly `target` records (bisection on length)"""
    lo, hi = 500, len(seq)
    assert n_records(ctx, head + [seq], kw) >= target
    while lo < hi:
        mid = (lo + hi) // 2
        if n_records(ctx, head + [seq[:mid]], kw) >= target:
            hi = mid
        else:
            lo = mid + 1
    out = head + [seq[:lo]]
    assert n_records(ctx, out, kw) == target, "record count %d not reachable" % target
    return out


def unrelated(ctx, rng, n, other, kw):
    """n random bases none of whose seed k-mers occurs in `other` (a seed-sized share of a random stretch would still
    match some: both sides keep only the low-hash k-mers)"""
    import skani_b200 as sk
    s = rand_seq(rng, n)
    for _ in range(10):
        e = sk.sketch_sequences(ctx, [[s]], sk.sketch_params(**kw)).export(0)
        hit = np.isin(e["kmer"], other)
        if not hit.any():
            return s
        for p in e["pos"][hit].astype(np.int64):                  # redraw every base of any window that holds p
            s[max(p - 15, 0):p + 16] = rand_seq(rng, len(s[max(p - 15, 0):p + 16]))
    raise AssertionError("could not remove the shared k-mers")


def test_tile_aligned_query_genomes_and_chunk_bound(ctx):
    import skani_b200 as sk
    kw = dict(c=125, k=15, marker_c=1000)
    rng = np.random.default_rng(17)
    R = rand_seq(rng, 1_500_000)                                     # slot 0: the ref role of every pair
    rk = sk.sketch_sequences(ctx, [[R]], sk.sketch_params(**kw)).export(0)["kmer"]
    rel = lambda a, b: mutate(rng, R[a:b], 0.01)                     # noqa: E731
    genomes = [[R]]
    names = {}
    for target in (1024, 1023, 1025, 2048):                           # one contig of exactly `target` records
        names[len(genomes)] = "n_rec=%d" % target
        genomes.append(cut_to_records(ctx, [], rel(10_000 * target // 1024, 400_000), target, kw))
    names[len(genomes)] = "contig boundary on a tile boundary"       # first contig: exactly one tile of records
    first = cut_to_records(ctx, [], rel(500_000, 700_000), TILE, kw)
    genomes.append(first + [rel(700_000, 850_000)])
    gap = len(genomes)
    names[gap] = "anchor-free tiles"                                 # 40 kb related, 450 kb unrelated, 80 kb related
    genomes.append([np.concatenate([rel(900_000, 940_000), unrelated(ctx, rng, 450_000, rk, kw), rel(1_000_000, 1_080_000)])])
    last = len(genomes)
    names[last] = "anchors only in the last, partial tile"
    genomes.append([np.concatenate([unrelated(ctx, rng, 260_000, rk, kw), rel(1_100_000, 1_112_000)])])
    bound = len(genomes)
    names[bound] = "chunk-staging bound reached"                     # contigs of m * 20 kb + 5 kb, related end to end
    genomes.append([mutate(rng, R[a:a + L], 0.002) for a, L in ((1_200_000, 65_000), (1_270_000, 105_000), (1_380_000, 25_000))])
    gs, osk = make_sets(ctx, genomes, kw)
    q = list(range(1, len(genomes)))
    pairs = [(0, g) for g in q] + [(g, 0) for g in q] + [(gap, last), (bound, 1)]
    gds = check_batch(ctx, gs, osk, pairs)
    by = {p: gd for p, gd in zip(pairs, gds)}
    for g in q:
        gd = by[(0, g)]
        assert roles(gd, 0, g) == (g, 0), names[g]
        assert len(gd["anchors"]) > 0, names[g]
    assert [gs.info(g)["n_records"] for g in (1, 2, 3, 4)] == [1024, 1023, 1025, 2048]
    e = gs.export(5)
    assert gs.info(5)["n_contigs"] == 2 and int(np.sum((e["cc"] >> 1) == 0)) == TILE
    assert np.any(by[(0, 5)]["anchors"][:, 0] == 1)                 # the second contig has anchors too
    # two or more whole tiles without anchors, then a catch-up singleton chunk on the far side
    eg = gs.export(gap)
    per_tile, _, _ = tile_stats(eg, by[(0, gap)]["anchors"])
    zero_run = max(len(s) for s in "".join("0" if x == 0 else "1" for x in per_tile).split("1"))
    assert zero_run >= 2, per_tile
    an, cf = by[(0, gap)]["anchors"], by[(0, gap)]["chunk_first"]
    sizes = np.diff(cf.astype(np.int64))
    assert np.any((sizes == 1) & (an[cf[:-1], 1] > 490_000)), "no catch-up singleton chunk after the gap"
    # all anchors in the last, partial tile
    el = gs.export(last)
    n = len(el["pos"])
    assert n % TILE != 0
    ri = record_index(el, by[(0, last)]["anchors"])
    assert len(ri) > 0 and ri.min() >= (n // TILE) * TILE
    # the pair's chunk count equals the staging slice's size, sum over contigs of ceil(len / 20 kb)
    lens = gs.export(bound)["contig_lengths"].astype(np.int64)
    max_chunks = int(np.sum((lens + 19_999) // 20_000))
    assert max_chunks == 4 + 6 + 2
    assert len(by[(0, bound)]["chunk_first"]) - 1 == max_chunks


# ---------------------------------------------------------------------------------------------------------------------
# 5. every DP variant, and the band the DP cannot hold
# ---------------------------------------------------------------------------------------------------------------------
# c -> band 2500 // c -> kernel (chain.cu run_batch): band <= 24 takes dp_group_kernel with GL lanes x NE candidates, FULLBAND
# (no band test) when band == GL * NE, with the 25-block register cap unless SK_DP_MINB=1; larger bands take
# dp_warp_kernel<NB> with NB >= band / 32 + 2 register sets.
@pytest.mark.parametrize("c,env", [(90, {}), (20, {}), (10, {}), (6, {}), (125, {}), (125, {"SK_DP_WARP": "1"}),
                                   (125, {"SK_DP_MINB": "1"}), (110, {"SK_DP_MINB": "1"}), (104, {}), (104, {"SK_DP_GL": "8"})],
                         ids=["c90_warp2", "c20_warp8", "c10_warp16", "c6_warp16_band416", "c125_gl4_ne5_fullband_cap25",
                              "c125_dp_warp2", "c125_gl4_ne5_fullband_uncapped", "c110_gl4_ne6", "c104_gl4_ne6_fullband_cap25",
                              "c104_gl8_ne3_fullband_cap25"])
def test_dp_variants_bit_exact(ctx, monkeypatch, c, env):
    for k, v in env.items():
        monkeypatch.setenv(k, v)
    genomes = synth_genomes(4, 300_000 if c < 30 else 500_000, 2)
    kw = dict(c=c, k=15, marker_c=max(c, 200) if c < 100 else 1000)
    gs, osk = make_sets(ctx, genomes, kw)
    gds = check_batch(ctx, gs, osk, [(0, 1), (1, 0), (2, 3), (0, 0)])
    assert all(len(gd["intervals"]) > 5 for gd in gds[:3])


def test_band_beyond_dp_is_refused_before_launch(ctx):
    import skani_b200 as sk
    genomes = synth_genomes(2, 200_000, 2)
    g5 = sk.sketch_sequences(ctx, genomes, sk.sketch_params(c=5, k=15, marker_c=200))
    before = ctx.launches
    with pytest.raises(sk.host.SkaniError, match="band > 479"):
        sk.chain_pairs(ctx, g5, g5, pair_ids([(0, 1)]))
    assert ctx.launches == before                                   # nothing ran
    gs, osk = make_sets(ctx, genomes, dict(c=125, k=15, marker_c=1000))
    check_batch(ctx, gs, osk, [(0, 1), (1, 0)])                     # the context still chains correctly


# ---------------------------------------------------------------------------------------------------------------------
# 6. the 2^20-record probe threshold: hash table (20-bit group start) just below it, bucket search at it
# ---------------------------------------------------------------------------------------------------------------------
def test_probe_threshold_2_pow_20_records(ctx):
    import skani_b200 as sk
    kw = dict(c=10, k=15, marker_c=200)
    rng = np.random.default_rng(23)
    seq = rand_seq(rng, 11_000_000)
    genomes = []
    for target in ((1 << 20) - 1, 1 << 20):
        g = cut_to_records(ctx, [], seq, target, kw)
        # the query: 600 kb around the record with the largest k-mer (the last group of the sorted ref-role view)
        e = sk.sketch_sequences(ctx, [g], sk.sketch_params(**kw)).export(0)
        p = int(e["pos"][int(np.argmax(e["kmer"]))])
        a = max(0, p - 300_000)
        qs = mutate(rng, g[0][a:a + 600_000], 0.01)
        qs[p - a - 50:p - a + 50] = g[0][p - 50:p + 50]
        genomes += [g, [qs]]
    gs, osk = make_sets(ctx, genomes, kw)
    assert [gs.info(i)["n_records"] for i in (0, 2)] == [(1 << 20) - 1, 1 << 20]
    gds = check_batch(ctx, gs, osk, [(0, 1), (2, 3), (1, 0)])
    for i, gd in ((0, gds[0]), (2, gds[1])):
        assert roles(gd, i, i + 1) == (i + 1, i)
        kr, kq = gs.export(i)["kmer"], gs.export(i + 1)["kmer"]
        assert kr.max() in set(kq.tolist())                          # the query hits the last k-mer group
        assert len(gd["anchors"]) > 10_000


# ---------------------------------------------------------------------------------------------------------------------
# 7. more than one batch of pairs, the later batch reusing the first one's (larger) buffers
# ---------------------------------------------------------------------------------------------------------------------
def test_pair_list_crossing_the_batch_limit(ctx):
    import skani_b200 as sk
    rng = np.random.default_rng(31)
    genomes = []
    for cl in range(3):                                               # 3 clusters of 90 related 5-8 kb genomes
        base = rand_seq(rng, 12_000)
        for i in range(90):
            a = int(rng.integers(0, 4_000))
            L = int(rng.integers(5_000, 8_000))
            genomes.append([mutate(rng, base[a:a + L], 0.01 + 0.02 * rng.random())])
    kw = dict(c=30, k=15, marker_c=200)
    gs, osk = make_sets(ctx, genomes, kw)
    n = len(genomes)
    size = np.array([gs.info(g)["n_records"] for g in range(n)], np.int64)
    pairs = [(r, q) for r in range(n) for q in range(n) if r != q]
    pairs.sort(key=lambda p: -(size[p[0]] + size[p[1]]))              # the largest pairs in the first batch
    assert len(pairs) > MAX_PAIRS_PER_BATCH
    ids = pair_ids(pairs)
    res = sk.chain_pairs(ctx, gs, gs, ids, as_array=True)
    n_hit = 0
    for i, (r, q) in enumerate(pairs):
        o = O.chain(osk[r], osk[q])
        assert (int(res[i]["ref_id"]), int(res[i]["query_id"])) == (r, q)
        if np.isnan(o.ani):
            assert np.isnan(res[i]["ani"]), (r, q)
            continue
        n_hit += 1
        for f in ("ani", "af_ref", "af_query"):
            assert abs(float(res[i][f]) - getattr(o, f)) <= TOL, (r, q, f)
    assert n_hit > len(pairs) // 5
    sample = sorted(set(rng.choice(MAX_PAIRS_PER_BATCH, 40, replace=False).tolist()) |
                    set(range(MAX_PAIRS_PER_BATCH - 3, MAX_PAIRS_PER_BATCH + 40)) |
                    set(rng.choice(np.arange(MAX_PAIRS_PER_BATCH, len(pairs)), 120, replace=False).tolist()) | {len(pairs) - 1})
    gds = sk.chain_pairs_debug(ctx, gs, gs, ids, sk.map_params(), keep=sample)
    for i in sample:
        r, q = pairs[i]
        assert bytes(gds[i]["result"]) == res[i].tobytes()
        assert_pair_equal(gds[i], O.chain_debug(osk[r], osk[q]))
    assert sum(len(gds[i]["anchors"]) > 0 for i in sample if i >= MAX_PAIRS_PER_BATCH) > 10
    assert_result_close(gds[sample[-1]]["result"], O.chain(osk[pairs[-1][0]], osk[pairs[-1][1]]))
