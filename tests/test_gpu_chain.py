"""GPU parity: screen + chain kernels vs the CPU oracle through the C ABI.  Integer stages (anchors, chunks, DP
scores/pointers, chain intervals, greedy selection, per-chunk weights) must be bit-exact; ANI/AF floats within 1e-4
(BASELINE.json north_star), in practice identical to the last f32 digit."""
import os

import numpy as np
import pytest

import oracle_py as O
from bench_support import synth
from fasta_py import read_fastx

pytestmark = pytest.mark.gpu
GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
TOL = 1e-4


@pytest.fixture(scope="module")
def ctx():
    import skani_b200 as sk
    c = sk.Context(0)
    yield c
    c.close()


def f2(x):
    return "%.2f" % float(np.float32(x) * np.float32(100.0))


def assert_result_close(g, o, tol=TOL):
    if np.isnan(o.ani):
        assert np.isnan(g.ani)
        return
    for f in ("ani", "af_query", "af_ref", "std", "ci_lower", "ci_upper"):
        assert abs(getattr(g, f) - getattr(o, f)) <= tol, (f, getattr(g, f), getattr(o, f))
    for f in ("q90_q", "q90_r", "q50_q", "q50_r", "q10_q", "q10_r", "num_contigs_q", "num_contigs_r",
              "avg_chain_int_len", "total_bases_covered"):
        assert getattr(g, f) == getattr(o, f), (f, getattr(g, f), getattr(o, f))


def assert_debug_equal(gd, od):
    assert gd["switched"] == od["switched"]
    assert np.array_equal(gd["anchors"], od["anchors"]), "anchors"
    assert np.array_equal(gd["chunk_first"], od["chunk_first"]), "chunk_first"
    assert np.array_equal(gd["chunk_nseeds"], od["chunk_nseeds"]), "chunk_nseeds"
    assert np.array_equal(gd["score"], od["score"]), "score"
    assert np.array_equal(gd["pointer"], od["pointer"]), "pointer"
    assert np.array_equal(gd["intervals"], od["intervals"]), "intervals"
    assert np.array_equal(gd["weight"], od["weight"]), "weights"
    assert np.allclose(gd["est"], od["est"], rtol=0, atol=1e-12), "ests"
    assert_result_close(gd["result"], od["result"])


def make_sets(ctx, genomes, sp_kw, individual=False):
    """genomes: list of lists of contig byte arrays -> (gpu set, [oracle sketches])"""
    import skani_b200 as sk
    gs = sk.sketch_sequences(ctx, genomes, sk.sketch_params(**sp_kw), individual_contig=individual)
    osk = []
    for gi, ctgs in enumerate(genomes):
        kept = [c for c in ctgs if len(c) >= 500]
        if not kept:
            continue
        if individual:
            for j, c in enumerate(kept):
                osk.append(O.sketch_from_contigs("g%06d" % gi, [c], **sp_kw))
        else:
            osk.append(O.sketch_from_contigs("g%06d" % gi, kept, **sp_kw))
    assert len(gs) == len(osk)
    return gs, osk


def synth_genomes(n, L, G):
    bases, off, goc = synth.generate(0, n, L, G=G)
    out = []
    for g in range(n):
        idx = np.nonzero(goc == g)[0]
        out.append([bases[int(off[i]):int(off[i + 1])] for i in idx])
    return out


@pytest.mark.parametrize("c,mc,learned", [(125, 1000, True), (30, 200, False), (200, 1000, True)])
def test_chain_debug_parity_synthetic(ctx, c, mc, learned):
    import skani_b200 as sk
    genomes = synth_genomes(8, 700_000, 4)
    kw = dict(c=c, k=15, marker_c=mc)
    gs, osk = make_sets(ctx, genomes, kw)
    mp = sk.map_params(learned_ani=learned)
    ocp = O.cmd(learned_ani=learned)
    for (r, q) in [(0, 1), (0, 2), (1, 3), (2, 3), (5, 6), (4, 7), (0, 5), (3, 3)]:
        gd = sk.chain_pair_debug(ctx, gs, gs, r, q, mp)
        od = O.chain_debug(osk[r], osk[q], ocp)
        assert_debug_equal(gd, od)


@pytest.mark.parametrize("lanes", ["4", "8"])
def test_chain_debug_parity_dp_lane_groups(ctx, monkeypatch, lanes):
    """The banded DP with 4 lanes per chunk / 8 chunks per warp (the default) and with 8
    lanes / 4 chunks per warp (SK_DP_GL=8) are both held to bit-exact per-anchor score / pointer / interval parity."""
    import skani_b200 as sk
    monkeypatch.setenv("SK_DP_GL", lanes)
    genomes = synth_genomes(8, 700_000, 4)
    for c in (125, 200, 110):          # band 20 / 12 (5 candidates per lane with 4 lanes), band 22 (6 candidates)
        gs, osk = make_sets(ctx, genomes, dict(c=c, k=15, marker_c=1000))
        for (r, q) in [(0, 1), (1, 3), (5, 6), (4, 7), (3, 3)]:
            assert_debug_equal(sk.chain_pair_debug(ctx, gs, gs, r, q, sk.map_params()), O.chain_debug(osk[r], osk[q], O.cmd()))


def test_triangle_parity_synthetic(ctx):
    import skani_b200 as sk
    n, L, G = 24, 400_000, 6
    bases, off, goc = synth.generate(0, n, L, G=G)
    res, st = sk.triangle(ctx, bases, off, goc, n)
    genomes = [[bases[int(off[i]):int(off[i + 1])] for i in np.nonzero(goc == g)[0]] for g in range(n)]
    osk = [O.sketch_from_contigs("g%06d" % g, genomes[g]) for g in range(n)]
    ores, info = O.triangle(osk, O.cmd())
    assert st.n_pairs_screened == info["n_chained"]
    got = {(r.ref_id, r.query_id): r for r in res}
    exp = {(r.ref_id, r.query_id): r for r in ores}
    assert set(got) == set(exp) and len(got) == n // G * (G * (G - 1) // 2)
    for key in exp:
        assert_result_close(got[key], exp[key])
    # screen alone
    gs = sk.sketch_contigs(ctx, bases, off, goc, n)
    pairs = sk.screen_triangle(ctx, gs)
    ro, cols = O.screen_triangle(osk)
    exp_pairs = [(i << 32) | int(j) for i in range(n) for j in cols[int(ro[i]):int(ro[i + 1])]]
    assert pairs.tolist() == sorted(exp_pairs)


def load_genome(name):
    return [np.frombuffer(s, np.uint8) for _, s in read_fastx(os.path.join(GOLD, name))]


def test_config1_ecoli_dist(ctx):
    """BASELINE.json configs[0]: skani dist refs/e.coli-EC590.fasta refs/e.coli-K12.fasta (query = EC590, ref = K12)."""
    import skani_b200 as sk
    k12, ec = load_genome("e.coli-K12.fasta.gz"), load_genome("e.coli-EC590.fasta.gz")
    for c, exp in [(125, ("99.39", "91.89", "92.46")), (200, ("99.42", "94.47", "95.06"))]:   # G13 / G4 goldens
        kw = dict(c=c, k=15, marker_c=1000)
        refs, oref = make_sets(ctx, [k12], kw)
        qs, oq = make_sets(ctx, [ec], kw)
        import ctypes
        qs.ctx.check(qs.ctx.L.sk_sketch_set_set_name_ranks(qs.h, np.array([0], np.uint64).ctypes.data))
        refs.ctx.check(refs.ctx.L.sk_sketch_set_set_name_ranks(refs.h, np.array([1], np.uint64).ctypes.data))
        pairs = sk.host.screen_query_ref(ctx, refs, qs, sk.map_params(), mode=0)
        assert pairs.tolist() == [0]
        gd = sk.chain_pair_debug(ctx, refs, qs, 0, 0, sk.map_params())
        oref[0]  # oracle names: ref "g000000" == query "g000000": tie-break not reached (scores differ)
        od = O.chain_debug(oref[0], oq[0], O.cmd())
        assert_debug_equal(gd, od)
        r = gd["result"]
        assert (f2(r.ani), f2(r.af_ref), f2(r.af_query)) == exp


def test_reads_vs_genome_g8_golden(ctx):
    """G8: dist --qi --robust, 364 ONT reads vs EC590 -> the reference's own 269 rows (test_results_versions/0.3.0:153-421)."""
    import skani_b200 as sk
    gold = {}
    for ln in open(os.path.join(GOLD, "g8_dist_qi_robust.tsv")):
        if not ln.startswith("#"):
            ani, afr, afq, name = ln.rstrip("\n").split("\t")
            gold[name] = (ani, afr, afq)
    recs = [(n, s) for n, s in read_fastx(os.path.join(GOLD, "o157_reads.fa.gz")) if len(s) >= 500]
    reads = [np.frombuffer(s, np.uint8) for _, s in recs]
    kw = dict(c=125, k=15, marker_c=1000)
    refs, _ = make_sets(ctx, [load_genome("e.coli-EC590.fasta.gz")], kw)
    qs = sk.sketch_sequences(ctx, [reads], sk.sketch_params(**kw), individual_contig=True)
    assert len(qs) == 364
    mp = sk.map_params(robust=True, learned_ani=False)
    pairs = sk.host.screen_query_ref(ctx, refs, qs, mp, mode=2)        # --qi => marker index on
    res = sk.chain_pairs(ctx, refs, qs, pairs, mp)
    got = {recs[r.query_id][0]: (f2(r.ani), f2(r.af_ref), f2(r.af_query)) for r in res if r.ani > 0.1}
    assert len(got) == 269
    assert got == gold


def test_small_genomes_viruses(ctx):
    import skani_b200 as sk
    recs = read_fastx(os.path.join(GOLD, "viruses.fna"))
    ctgs = [np.frombuffer(s, np.uint8) for _, s in recs]
    for kw, rescue in [(dict(c=125, k=15, marker_c=1000), True), (dict(c=30, k=15, marker_c=200), False)]:
        gs, osk = make_sets(ctx, [ctgs], kw, individual=True)
        mp = sk.map_params(learned_ani=False, rescue_small=rescue)
        pairs = sk.screen_triangle(ctx, gs, mp)
        ro, cols = O.screen_triangle(osk, rescue_small=rescue)
        assert pairs.tolist() == sorted((i << 32) | int(j) for i in range(3) for j in cols[int(ro[i]):int(ro[i + 1])])
        res = sk.chain_pairs(ctx, gs, gs, pairs, mp)
        for r in res:
            o = O.chain(osk[r.ref_id], osk[r.query_id], O.cmd(learned_ani=False, rescue_small=rescue))
            assert_result_close(r, o)
            gd = sk.chain_pair_debug(ctx, gs, gs, r.ref_id, r.query_id, mp)
            assert_debug_equal(gd, O.chain_debug(osk[r.ref_id], osk[r.query_id], O.cmd(learned_ani=False, rescue_small=rescue)))


def test_bucket_probe_fallback_path(ctx, monkeypatch):
    """Genomes with >= 2^20 seed records use the bucket-index search instead of the per-genome hash table;
    SK_FORCE_BUCKET_PROBE forces that path so it stays covered."""
    import skani_b200 as sk
    monkeypatch.setenv("SK_FORCE_BUCKET_PROBE", "1")
    genomes = synth_genomes(4, 500_000, 4)
    kw = dict(c=125, k=15, marker_c=1000)
    gs, osk = make_sets(ctx, genomes, kw)
    for (r, q) in [(0, 1), (2, 3), (1, 2)]:
        assert_debug_equal(sk.chain_pair_debug(ctx, gs, gs, r, q, sk.map_params()), O.chain_debug(osk[r], osk[q], O.cmd()))


def test_large_multicontig_pair_global_fallbacks(ctx):
    """> 1024 chunks and > 1024 chain intervals per pair: the shared-memory sorts of select_kernel / final_kernel fall
    back to their global-memory paths (the MAG-sized pairs of the reference's fast_eukaryote_test)."""
    import skani_b200 as sk
    genomes = synth_genomes(3, 24_000_000, 3)          # member 2 is cut into 50 contigs, member 1 carries an inversion
    kw = dict(c=125, k=15, marker_c=1000)
    gs, osk = make_sets(ctx, genomes, kw)
    for (r, q) in [(0, 2), (1, 2), (0, 1)]:
        gd = sk.chain_pair_debug(ctx, gs, gs, r, q, sk.map_params())
        od = O.chain_debug(osk[r], osk[q], O.cmd())
        assert len(od["chunk_first"]) - 1 > 1024 and len(od["intervals"]) > 1024
        assert_debug_equal(gd, od)


@pytest.mark.parametrize("kw", [dict(robust=True), dict(median=True, learned_ani=False), dict(min_af=0.999), dict(both_min_af=0.999),
                                dict(min_af=-1.0), dict(learned_ani=False)])
def test_map_param_variants(ctx, kw):
    import skani_b200 as sk
    genomes = synth_genomes(6, 400_000, 3)
    gs, osk = make_sets(ctx, genomes, dict(c=125, k=15, marker_c=1000))
    mp, ocp = sk.map_params(**kw), O.cmd(**kw)
    pairs = [(0, 1), (0, 2), (1, 2), (3, 4), (0, 3), (2, 5)]      # incl. unrelated pairs (no anchors -> NaN)
    res = sk.chain_pairs(ctx, gs, gs, np.array([(r << 32) | q for r, q in pairs], np.uint64), mp)
    for (r, q), g in zip(pairs, res):
        assert (g.ref_id, g.query_id) == (r, q)
        assert_result_close(g, O.chain(osk[r], osk[q], ocp))


def test_degenerate_sets(ctx):
    import skani_b200 as sk
    # no pairs
    genomes = synth_genomes(2, 300_000, 1)               # two unrelated genomes: screen passes nothing
    gs, osk = make_sets(ctx, genomes, dict(c=125, k=15, marker_c=1000))
    assert len(sk.screen_triangle(ctx, gs)) == 0
    assert sk.chain_pairs(ctx, gs, gs, np.zeros(0, np.uint64)) == []
    r = sk.chain_pairs(ctx, gs, gs, np.array([1], np.uint64))[0]           # unrelated pair chained anyway: no anchors
    assert np.isnan(r.ani) and np.isnan(O.chain(osk[0], osk[1]).ani)
    # a single genome: triangle has no rows
    one = sk.sketch_sequences(ctx, [genomes[0]])
    assert len(sk.screen_triangle(ctx, one)) == 0
    # genome made of N only: sketch exists but is empty (reference: all_ns.fa -> 0 rows)
    ns = sk.sketch_sequences(ctx, [[np.full(2000, ord("N"), np.uint8)], genomes[0]])
    assert ns.info(0)["n_records"] == 0 and ns.info(0)["n_markers"] == 0
    assert len(sk.screen_triangle(ctx, ns, sk.map_params(rescue_small=False))) == 0
    pr = sk.screen_triangle(ctx, ns)                                        # rescue_small: < 20 markers passes everything
    assert pr.tolist() == [1]
    rr = sk.chain_pairs(ctx, ns, ns, pr)[0]
    assert np.isnan(rr.ani)


def test_chunk_catchup_after_long_gap(ctx):
    """Anchor-free stretches longer than a fragment (20 kb) make the reference's chunk loop emit singleton 'catch-up'
    chunks (src/chain.rs:744-793); those pairs take the general prefix-min kernel instead of the fast path."""
    import skani_b200 as sk
    rng = np.random.default_rng(7)
    base = synth_genomes(1, 900_000, 1)[0][0].copy()
    other = base.copy()
    for a, b in [(100_000, 190_000), (400_000, 465_000), (700_000, 724_000)]:     # 90 kb, 65 kb, 24 kb of unrelated sequence
        other[a:b] = rng.choice(np.frombuffer(b"ACGT", np.uint8), b - a)
    mut = rng.random(len(other)) < 0.01
    other[mut] = rng.choice(np.frombuffer(b"ACGT", np.uint8), int(mut.sum()))
    # a multi-contig variant as well: contig boundaries inside and outside the gaps
    cuts = [0, 150_000, 420_000, 430_000, 900_000]
    multi = [other[cuts[i]:cuts[i + 1]] for i in range(4)]
    kw = dict(c=125, k=15, marker_c=1000)
    gs, osk = make_sets(ctx, [[base], [other], multi], kw)
    for (r, q) in [(0, 1), (1, 0), (0, 2), (2, 0), (1, 2)]:
        gd = sk.chain_pair_debug(ctx, gs, gs, r, q, sk.map_params())
        od = O.chain_debug(osk[r], osk[q], O.cmd())
        assert_debug_equal(gd, od)
    sizes = np.diff(O.chain_debug(osk[0], osk[1], O.cmd())["chunk_first"])
    assert (sizes == 1).sum() >= 2          # the oracle really produced catch-up singleton chunks


def test_pipelined_triangle_equals_simple(ctx, monkeypatch):
    """sk_triangle's upload/seed || screen/chain software pipeline (used for >= 4 GiB inputs) gives the same result set."""
    import skani_b200 as sk
    n, L, G = 30, 300_000, 5
    bases, off, goc = synth.generate(0, n, L, G=G)
    monkeypatch.setenv("SK_NO_PIPELINE", "1")
    r0, st0 = sk.triangle(ctx, bases, off, goc, n, as_array=True)
    monkeypatch.delenv("SK_NO_PIPELINE")
    monkeypatch.setenv("SK_FORCE_PIPELINE", "1")
    r1, st1 = sk.triangle(ctx, bases, off, goc, n, as_array=True)
    assert st0.n_pairs_screened == st1.n_pairs_screened == n // G * (G * (G - 1) // 2)
    k0 = np.sort(r0, order=["ref_id", "query_id"]); k1 = np.sort(r1, order=["ref_id", "query_id"])
    assert len(k0) == len(k1) and k0.tobytes() == k1.tobytes()


def test_screen_triangle_block_partitions_the_pair_list(ctx):
    """sk_screen_triangle_block (one GPU's share of the sharded screen): for any cut of the genome range into blocks the union
    of the blocks' lists is sk_screen_triangle's list, each block holding exactly the pairs whose larger index it owns --
    including genomes with < 20 markers (rescue rows pass whole columns) and a genome without sequence."""
    import skani_b200 as sk
    L, G = 200_000, 3
    b0, off0, goc0 = synth.generate(0, 12, L, G=G)
    contigs, goc = [], []
    real = iter(range(12))
    n = 16
    for g in range(n):
        if g in (0, 6, 13):
            contigs.append(b0[int(off0[0]) + 1500 * g: int(off0[0]) + 1500 * g + 7000].copy()); goc.append(g)
        elif g == 9:
            continue                                                   # no contigs: empty sketch
        else:
            r = next(real)
            for i in np.nonzero(goc0 == r)[0]:
                contigs.append(b0[int(off0[i]):int(off0[i + 1])]); goc.append(g)
    bases = np.concatenate(contigs)
    off = np.concatenate([[0], np.cumsum([len(c) for c in contigs])]).astype(np.uint64)
    sset = sk.sketch_contigs(ctx, bases, off, np.asarray(goc, np.uint32), n)
    full = sk.screen_triangle(ctx, sset)
    assert len(full) > 20
    for cuts in ([0, n], [0, 5, n], [0, 1, 2, 9, 10, n], [0, 0, 7, 7, n]):
        parts = [sk.screen_triangle_block(ctx, sset, cuts[i], cuts[i + 1]) for i in range(len(cuts) - 1)]
        for i, p in enumerate(parts):
            j = (p & np.uint64(0xFFFFFFFF)).astype(np.int64)
            assert np.all((j >= cuts[i]) & (j < cuts[i + 1])) and np.all(np.diff(p.astype(np.int64)) > 0)
        assert np.array_equal(np.sort(np.concatenate(parts)), full)
    import os
    os.environ["SK_FULL_RESCREEN"] = "1"                               # the fallback (one-shot screen + filter) gives the same blocks
    try:
        fb = sk.screen_triangle_block(ctx, sset, 5, n)
    finally:
        del os.environ["SK_FULL_RESCREEN"]
    assert np.array_equal(fb, sk.screen_triangle_block(ctx, sset, 5, n))
    sset.free()


@pytest.mark.parametrize("pipelined", [False, True])
def test_triangle_on_device_resident_bases(ctx, monkeypatch, pipelined):
    """sk_triangle / sk_triangle_local on a DEVICE pointer (genomes already in HBM: the bench's `value` leg) give the result
    bytes of the host-buffer call, through the one-shot path and through the pipeline (several sub-batches and waves)."""
    import torch
    import skani_b200 as sk
    n, L, G = 20, 250_000, 4
    bases, off, goc = synth.generate(0, n, L, G=G)
    r0, st0 = sk.triangle(ctx, bases, off, goc, n, as_array=True)
    dev = torch.from_numpy(bases).cuda()
    if pipelined:
        monkeypatch.setenv("SK_FORCE_PIPELINE", "1")
        monkeypatch.setenv("SK_SUBBATCH_BYTES", "700000")
    r1, st1 = sk.triangle(ctx, int(dev.data_ptr()), off, goc, n, as_array=True)
    r2, kept, _ = sk.triangle_local(ctx, int(dev.data_ptr()), off, goc, n)
    assert len(kept) == n
    kept.free()
    k0 = np.sort(r0, order=["ref_id", "query_id"]).tobytes()
    assert len(r0) > 0 and k0 == np.sort(r1, order=["ref_id", "query_id"]).tobytes() == np.sort(r2, order=["ref_id", "query_id"]).tobytes()
    assert st0.n_pairs_screened == st1.n_pairs_screened


@pytest.mark.parametrize("rescreen", [False, True])
def test_pipelined_triangle_small_marker_sets(ctx, monkeypatch, rescreen):
    """Incremental screen of the pipelined triangle vs the one-shot screen when some genomes have < 20 markers (screen_refs'
    rescue rule is decided by the SMALLER index of a pair, src/screen.rs:158-160) or no markers at all, in every wave position."""
    import skani_b200 as sk
    L, G = 200_000, 3
    b0, off0, goc0 = synth.generate(0, 12, L, G=G)
    rng = np.random.default_rng(11)
    contigs, goc = [], []
    tiny_at = {0, 5, 9, 14}        # slots of tiny genomes (6 kb: ~6 markers) among the 12 real ones
    real = iter(range(12))
    n = 16
    for g in range(n):
        if g in tiny_at:
            src = b0[int(off0[0]) + 1000 * g: int(off0[0]) + 1000 * g + 6000].copy()     # related to genome 0's cluster
            contigs.append(src); goc.append(g)
        else:
            r = next(real)
            for i in np.nonzero(goc0 == r)[0]:
                contigs.append(b0[int(off0[i]):int(off0[i + 1])]); goc.append(g)
    bases = np.concatenate(contigs)
    off = np.concatenate([[0], np.cumsum([len(c) for c in contigs])]).astype(np.uint64)
    goc = np.asarray(goc, dtype=np.uint32)
    monkeypatch.setenv("SK_NO_PIPELINE", "1")
    r0, st0 = sk.triangle(ctx, bases, off, goc, n, as_array=True)
    monkeypatch.delenv("SK_NO_PIPELINE")
    monkeypatch.setenv("SK_FORCE_PIPELINE", "1")
    monkeypatch.setenv("SK_SUBBATCH_BYTES", "450000")
    if rescreen:
        monkeypatch.setenv("SK_FULL_RESCREEN", "1")
    r1, st1 = sk.triangle(ctx, bases, off, goc, n, as_array=True)
    assert st0.n_pairs_screened == st1.n_pairs_screened and st0.n_pairs_screened >= 4 * 8   # rescue rows pass whole columns
    k0 = np.sort(r0, order=["ref_id", "query_id"]); k1 = np.sort(r1, order=["ref_id", "query_id"])
    assert len(k0) == len(k1) and k0.tobytes() == k1.tobytes()


@pytest.mark.parametrize("subbatch", ["350000", "1300000", "2500000"])
def test_pipelined_triangle_many_uneven_waves_vs_oracle(ctx, monkeypatch, subbatch):
    """The pipelined path with several waves of uneven size (sub-batches of 1 / 4 / 8 genomes, wave threshold n/8), genomes
    WITHOUT sequence in the middle and at the end (empty sketches), a cluster cut by every wave boundary, shuffled genome
    order: the kept (ref, query, ANI, AF) set must equal the unpipelined result byte for byte AND the oracle within 1e-4."""
    import skani_b200 as sk
    n_real, L, G = 22, 300_000, 4
    ids = synth.shuffled_ids(n_real, 3)
    b0, off0, goc0 = synth.generate_ids(ids, L, G=G)
    # genome slots: real genomes 0..9, an empty genome (no contigs), real 10..21, two empty genomes at the end
    slot = np.concatenate([np.arange(10), np.arange(11, 23)])
    goc = slot[goc0].astype(np.uint32)
    n = 25
    monkeypatch.setenv("SK_NO_PIPELINE", "1")
    r0, _ = sk.triangle(ctx, b0, off0, goc, n, as_array=True)
    monkeypatch.delenv("SK_NO_PIPELINE")
    monkeypatch.setenv("SK_FORCE_PIPELINE", "1")
    monkeypatch.setenv("SK_SUBBATCH_BYTES", subbatch)
    r1, _ = sk.triangle(ctx, b0, off0, goc, n, as_array=True)
    k0 = np.sort(r0, order=["ref_id", "query_id"]); k1 = np.sort(r1, order=["ref_id", "query_id"])
    assert len(k0) == len(k1) > 0 and k0.tobytes() == k1.tobytes()
    osk = []
    for g in range(n):
        idx = np.nonzero(goc == g)[0]
        osk.append(O.sketch_from_contigs("g%06d" % g, [b0[int(off0[i]):int(off0[i + 1])] for i in idx]))
    ores, _ = O.triangle(osk, O.cmd())
    exp = {(r.ref_id, r.query_id): r for r in ores}
    got = {(int(r["ref_id"]), int(r["query_id"])): r for r in k1}
    assert set(got) == set(exp)
    for k, e in exp.items():
        for f in ("ani", "af_ref", "af_query"):
            assert abs(float(got[k][f]) - getattr(e, f)) <= TOL, (k, f)


def test_append_then_chain_parity(ctx):
    """sk_sketch_set_append (the merge the pipelined worker and database loaders rely on): chaining across the appended
    boundary gives the oracle's results, and user-set name ranks survive the append."""
    import skani_b200 as sk
    n, L, G = 8, 300_000, 4
    bases, off, goc = synth.generate(0, n, L, G=G)
    n3 = int(np.searchsorted(goc, 3))
    a = sk.sketch_contigs(ctx, bases[:3 * L], off[:n3 + 1], goc[:n3], 3)
    b = sk.sketch_contigs(ctx, bases[3 * L:], off[n3:] - off[n3], goc[n3:] - 3, n - 3)
    a.set_name_ranks(np.arange(3))
    a.append(b)
    assert len(a) == n
    pairs = sk.screen_triangle(ctx, a)
    res = sk.chain_pairs(ctx, a, a, pairs, as_array=True)
    osk = [O.sketch_from_contigs("g%06d" % g, [bases[int(off[i]):int(off[i + 1])] for i in np.nonzero(goc == g)[0]]) for g in range(n)]
    ores, _ = O.triangle(osk, O.cmd())
    exp = {(r.ref_id, r.query_id): r for r in ores}
    got = {(int(r["ref_id"]), int(r["query_id"])): r for r in res if r["ani"] > 0.1}
    assert set(got) == set(exp) and len(exp) == 2 * (G * (G - 1) // 2)
    for k, e in exp.items():
        for f in ("ani", "af_ref", "af_query"):
            assert abs(float(got[k][f]) - getattr(e, f)) <= TOL, (k, f)
