"""Pins the CPU oracle (oracle/) against the golden vectors / known-answer tests the reference holds for the hot path
(SURVEY.md section 8c) whose inputs are stored under tests/golden/ (see its README); the GPU tests compare the CUDA path
with the oracle pinned here."""
import os

import numpy as np

import oracle_py as O

GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")


def f2(x):
    """Rust `{:.2}` of an f32 product, as file_io.rs:83-96 prints it."""
    return "%.2f" % float(np.float32(x) * np.float32(100.0))


def p(name):
    return os.path.join(GOLD, name)


# G2: tests/tests.rs:130-144 -- AVX2 path == scalar path on the 120-base string, c = 10
def test_g2_avx2_equals_scalar():
    s = b"ATCAGATTTAAAAAAAAATTTTGCTAGCTGATCGATCGATCGATGTGTATATATTAAAAGAGAGAGAGGGGGGGGAAAAAAAAAAAAACTGATCGATCGATGCTAGCTAGTCAGTCGATG"
    assert len(s) == 120
    L = O.lib()
    buf = np.frombuffer(s, np.uint8)
    # the seeders are called directly (no MIN_LENGTH_CONTIG rule), as tests/tests.rs does
    a = O.Sketch(L.orc_seed_one_contig(buf.ctypes.data, len(s), 10, 15, 1000, 1))
    b = O.Sketch(L.orc_seed_one_contig(buf.ctypes.data, len(s), 10, 15, 1000, 0))
    ea, eb = a.export(), b.export()
    assert a.n_records > 0
    for key in ("kmer", "pos", "cc", "markers"):
        assert np.array_equal(ea[key], eb[key])


# G3: tests/tests.rs:149-157 -- 154 x 'N' + 'n', c = 30, scalar path -> zero seeds
def test_g3_all_n_scalar():
    s = b"N" * 154 + b"n"
    buf = np.frombuffer(s, np.uint8)
    a = O.Sketch(O.lib().orc_seed_one_contig(buf.ctypes.data, len(s), 30, 15, 1000, 0))
    assert a.n_kmers == 0


def test_g4_dist_fast_ec590_k12():
    # test_results_versions/0.3.0:121  (`dist EC590 K12 --fast -n 3`; first positional is the query)
    r, _ = O.sketch_files([p("e.coli-K12.fasta.gz")], c=200)
    q, _ = O.sketch_files([p("e.coli-EC590.fasta.gz")], c=200)
    res = O.dist(r, q, O.cmd(learned_ani=True))
    assert len(res) == 1
    assert (f2(res[0].ani), f2(res[0].af_ref), f2(res[0].af_query)) == ("99.42", "94.47", "95.06")


def test_g8_dist_qi_robust_269_rows():
    gold = {}
    for ln in open(os.path.join(GOLD, "g8_dist_qi_robust.tsv")):
        if ln.startswith("#"):
            continue
        ani, afr, afq, name = ln.rstrip("\n").split("\t")
        gold[name] = (ani, afr, afq)
    assert len(gold) == 269
    refs, _ = O.sketch_files([p("e.coli-EC590.fasta.gz")])
    qs, _ = O.sketch_files([p("o157_reads.fa.gz")], individual=True)
    assert len(qs) == 364
    # --qi: marker index on (parse.rs:750), learned ANI off (regression.rs:8-10), --robust
    res = O.dist(refs, qs, O.cmd(robust=True, learned_ani=False), use_index=True)
    got = {qs[r.query_id].contig_name(0): (f2(r.ani), f2(r.af_ref), f2(r.af_query)) for r in res}
    assert len(got) == 269
    assert got == gold


def test_g10_result_counts_on_reads():
    # test_results_versions/0.3.0:60-69, tests/int_test_new.rs:56-133
    reads = [p("o157_reads.fa.gz")]
    ind, _ = O.sketch_files(reads, individual=True)
    res, _ = O.triangle(ind, O.cmd(learned_ani=False, rescue_small=True))          # triangle -i -E
    assert len(res) == 270
    res, _ = O.triangle(ind, O.cmd(learned_ani=False, rescue_small=False))         # --faster-small
    assert len(res) == 154
    big, _ = O.sketch_files(reads, individual=True, marker_c=1000000)
    res, _ = O.triangle(big, O.cmd(learned_ani=False, screen_val=0.95))            # -s 95 -m 1000000
    assert len(res) == 345
    big2, _ = O.sketch_files(reads, individual=True, marker_c=10000000)
    res, _ = O.triangle(big2, O.cmd(learned_ani=False))                            # -m 10000000
    assert len(res) == 345
    ref, _ = O.sketch_files([p("e.coli-EC590.fasta.gz")])
    # dist --qi: index on
    assert len(O.dist(ref, ind, O.cmd(learned_ani=False, rescue_small=False), use_index=True)) == 175
    assert len(O.dist(ref, ind, O.cmd(learned_ani=False, rescue_small=True), use_index=True)) == 269
    assert len(O.dist(ref, ind, O.cmd(learned_ani=False, rescue_small=False, screen_val=0.95), use_index=True)) == 87
    refb, _ = O.sketch_files([p("e.coli-EC590.fasta.gz")], marker_c=10000000000)
    indb, _ = O.sketch_files(reads, individual=True, marker_c=10000000000)
    assert len(O.dist(refb, indb, O.cmd(learned_ani=False, rescue_small=False), use_index=True)) == 0


def test_g11_self_vs_self():
    # tests/tests.rs:43-60 chains E. coli W against itself; any complete genome has the property, K12 is the one stored here
    r, _ = O.sketch_files([p("e.coli-K12.fasta.gz")])
    res = O.chain(r[0], r[0], O.cmd(learned_ani=False))
    assert res.ani >= 1.0 and res.af_query >= 0.99 and res.af_ref >= 0.99  # tests/tests.rs:57-59


def test_g12_viruses_small_genomes():
    # tests/int_test_new.rs:58-81: row0 in (99.0, 99.9), row1 > 99.9, with and without --faster-small;
    # --small-genomes == -c 30 -m 200 --faster-small (parse.rs:847-853)
    for kw, cp in [(dict(), O.cmd(learned_ani=False)), (dict(), O.cmd(learned_ani=False, rescue_small=False)),
                   (dict(c=30, marker_c=200), O.cmd(learned_ani=False, rescue_small=False))]:
        sk, _ = O.sketch_files([p("viruses.fna")], individual=True, **kw)
        assert len(sk) == 3
        res, _ = O.triangle(sk, cp)
        got = {(r.ref_id, r.query_id): r.ani * 100 for r in res}
        assert set(got) == {(0, 1), (0, 2), (1, 2)}
        assert 99.0 < got[(0, 1)] < 99.9
        assert got[(0, 2)] > 99.9 and got[(1, 2)] > 99.9


def test_g13_readme_example_config1():
    # README.md:48,142 / BASELINE.json configs[0]: `skani dist refs/e.coli-EC590.fasta refs/e.coli-K12.fasta`
    r, _ = O.sketch_files([p("e.coli-K12.fasta.gz")])
    q, _ = O.sketch_files([p("e.coli-EC590.fasta.gz")])
    res = O.dist(r, q, O.cmd(learned_ani=True))
    assert (f2(res[0].ani), f2(res[0].af_ref), f2(res[0].af_query)) == ("99.39", "91.89", "92.46")


def test_degenerate_inputs():
    # tests/int_test_new.rs:135-163: missing file, non-FASTA, all < 500 bp, all-N produce no sketches / no rows
    sk, nwarn = O.sketch_files([p("does_not_exist.fa"), p("list.txt"), p("test.fasta"), p("empty_fasta.fa")])
    assert len(sk) == 0 and nwarn == 4
    sk, _ = O.sketch_files([p("all_ns.fa")])
    assert len(sk) == 1 and sk[0].n_records == 0 and sk[0].n_markers == 0
    res, _ = O.triangle(sk + sk, O.cmd())
    assert len(res) == 0
