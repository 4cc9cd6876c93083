"""GPU: `skani-b200 sketch` writes a skani v0.3.0 database whose content (decoded by the independent Python decoder) is
bit-identical to the oracle's sketches, and `skani-b200 search` on it reproduces the oracle's search rows (no test pins
the oracle's search to the reference's golden G7; tests/test_oracle_goldens.py covers G2-G4, G8 and G10-G13).  Covers the consolidated database, the
--separate-sketches layout, FASTA queries and .sketch queries (src/sketch.rs, src/search.rs, src/sketch_db.rs)."""
import os
import subprocess

import numpy as np
import pytest

import oracle_py as O
import skani_db_py as D

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
BIN = os.path.join(ROOT, "skani_b200", "skani-b200")
GOLD = os.path.join(ROOT, "tests", "golden")
FILES = [os.path.join(GOLD, f) for f in ("e.coli-K12.fasta.gz", "viruses.fna", "e.coli-EC590.fasta.gz")]


def f2(x):
    return "%.2f" % float(np.float32(x) * np.float32(100.0))


def run(args):
    p = subprocess.run([BIN] + args, capture_output=True, text=True, timeout=600)
    assert p.returncode == 0, p.stderr
    return p.stdout


def check_against_oracle(decoded, osk):
    e = osk.export()
    assert decoded["file_name"] == osk.file_name
    assert decoded["records"] == list(zip(e["kmer"].tolist(), e["pos"].tolist(), e["cc"].tolist()))
    assert decoded["n_keys"] == osk.n_kmers
    assert decoded["markers"] == e["markers"].tolist()
    assert decoded["contig_lengths"] == e["contig_lengths"].tolist()
    assert decoded["contigs"] == [osk.contig_name(i) for i in range(osk.n_contigs)]
    assert decoded["total_len"] == osk.total_len and (decoded["marker_c"], decoded["c"], decoded["k"]) == (125, 125, 15)


def rows_of(out):
    lines = out.strip().split("\n")
    assert lines[0].startswith("Ref_file\tQuery_file\tANI\tAlign_fraction_ref\tAlign_fraction_query\tRef_name\tQuery_name")
    return sorted(tuple(ln.split("\t")[:7]) for ln in lines[1:])


def test_sketch_then_search(tmp_path):
    osk, _ = O.sketch_files(FILES)                      # sorted by file name, like the database
    db = str(tmp_path / "db")
    run(["sketch"] + FILES + ["-o", db])
    par, sk, mk, index = D.read_db(db)
    assert (par["c"], par["k"], par["marker_c"]) == (125, 15, 1000)
    assert open(os.path.join(db, "markers.bin"), "rb").read(626) == D.expected_params_bytes(125, 15, 1000)
    assert [s["file_name"] for s in sk] == [m["file_name"] for m in mk] == [i[0] for i in index] == sorted(FILES)
    for s, m, o in zip(sk, mk, osk):
        check_against_oracle(s, o)
        assert m["markers"] == s["markers"] and not m["has_seeds"] and m["contigs"] == s["contigs"]
    # an existing output directory is refused (src/sketch.rs:19-22)
    p = subprocess.run([BIN, "sketch", FILES[0], "-o", db], capture_output=True, text=True)
    assert p.returncode == 1 and "Output directory exists" in p.stderr

    # ---- search: EC590 (FASTA query) against the database; expected rows from the oracle's search
    q, _ = O.sketch_files([FILES[2]])
    exp = O.search(osk, q, O.cmd(learned_ani=True, min_af=-1.0, rescue_small=False))
    want = sorted((osk[r.ref_id].file_name, q[r.query_id].file_name, f2(r.ani), f2(r.af_ref), f2(r.af_query),
                   osk[r.ref_id].contig_name(0), q[r.query_id].contig_name(0)) for r in exp)
    assert len(want) == 2                               # itself and K12; the viruses fail the marker screen
    got = rows_of(run(["search", "-d", db, FILES[2]]))
    assert got == want
    assert ("100.00", "100.00", "100.00") in [g[2:5] for g in got]
    # -n 1 keeps the best hit per query; --median / --no-learned-ani follow the oracle too
    assert rows_of(run(["search", "-d", db, FILES[2], "-n", "1"])) == [w for w in want if w[2] == "100.00"]
    exp_m = O.search(osk, q, O.cmd(median=True, learned_ani=False, min_af=-1.0, rescue_small=False))
    want_m = sorted((osk[r.ref_id].file_name, q[r.query_id].file_name, f2(r.ani), f2(r.af_ref), f2(r.af_query),
                     osk[r.ref_id].contig_name(0), q[r.query_id].contig_name(0)) for r in exp_m)
    assert rows_of(run(["search", "-d", db, FILES[2], "--median"])) == want_m

    # ---- --separate-sketches layout: same sketches, searchable, and its .sketch files work as queries
    sep = str(tmp_path / "sep")
    run(["sketch"] + FILES + ["-o", sep, "--separate-sketches"])
    for f, o in zip(sorted(FILES), osk):
        b = open(os.path.join(sep, os.path.basename(f) + ".sketch"), "rb").read()
        c = D.Cur(b)
        assert D.params(c)["c"] == 125
        check_against_oracle(D.sketch(c), o)
        assert c.o == len(b)
    assert rows_of(run(["search", "-d", sep, FILES[2]])) == want
    assert rows_of(run(["search", "-d", db, os.path.join(sep, "e.coli-EC590.fasta.gz.sketch")])) == want

    # ---- per-record queries (--qi) against the database: the three virus records find themselves / each other
    qi, _ = O.sketch_files([FILES[1]], individual=True)
    exp_i = O.search(osk, qi, O.cmd(learned_ani=False, min_af=-1.0, rescue_small=False), use_index=True)
    want_i = sorted((osk[r.ref_id].file_name, qi[r.query_id].file_name, f2(r.ani), f2(r.af_ref), f2(r.af_query),
                     osk[r.ref_id].contig_name(0), qi[r.query_id].contig_name(0)) for r in exp_i)
    assert rows_of(run(["search", "-d", db, FILES[1], "--qi"])) == want_i
    # results appended in query blocks (INTERMEDIATE_WRITE_COUNT, src/search.rs:255-279): same rows with a block size of 1
    env = dict(os.environ, SK_INTERMEDIATE_WRITE_COUNT="1")
    p = subprocess.run([BIN, "search", "-d", db, FILES[1], "--qi"], capture_output=True, text=True, timeout=600, env=env)
    assert p.returncode == 0 and rows_of(p.stdout) == want_i and "INFO Writing results for 1 query sequences." in p.stderr


def test_sketch_files_as_dist_and_triangle_inputs(tmp_path):
    """.sketch files instead of FASTA (refs_are_sketch / queries_are_sketch, src/dist.rs:17-50, src/triangle.rs:16-24): the
    reference's golden G8 with its literal argument shape `dist -r EC590.sketch markers.bin -q reads --qi --robust`
    (test_results_versions/0.3.0:153-421), and triangle over a sketch folder == triangle over the FASTA files."""
    sep = str(tmp_path / "sep")
    run(["sketch"] + FILES + ["-o", sep, "--separate-sketches"])
    gold = {}
    for ln in open(os.path.join(GOLD, "g8_dist_qi_robust.tsv")):
        if not ln.startswith("#"):
            ani, afr, afq, name = ln.rstrip("\n").split("\t")
            gold[name] = (ani, afr, afq)
    out = run(["dist", "-r", os.path.join(sep, "e.coli-EC590.fasta.gz.sketch"), os.path.join(sep, "markers.bin"),
               "-q", os.path.join(GOLD, "o157_reads.fa.gz"), "--qi", "--robust"])
    rows = [ln.split("\t") for ln in out.strip().split("\n")[1:]]
    assert len(rows) == 269 and {r[6]: (r[2], r[3], r[4]) for r in rows} == gold
    assert all(r[0] == sorted(FILES)[0] for r in rows)            # Ref_file = the name stored in the sketch
    sk_files = [os.path.join(sep, os.path.basename(f) + ".sketch") for f in FILES]
    assert rows_of(run(["triangle", "-E"] + sk_files + [os.path.join(sep, "markers.bin")])) == rows_of(run(["triangle", "-E"] + FILES))
    both = rows_of(run(["dist", "-q", sk_files[2], "-r", sk_files[0]]))           # query EC590, ref K12: README pair (G13)
    assert [b[2:5] for b in both] == [("99.39", "91.89", "92.46")]
