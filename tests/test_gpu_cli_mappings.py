"""`--mappings FILE` on dist, search and triangle: the main output is byte-identical with and without it, the file holds
exactly the printed pairs in their order, its intervals lie inside their contigs, it does not depend on the input type, the
number of GPUs or the write blocks, and on a planted pair it finds the planted segments on the right strand.  Unsupported
paths are refused."""
import os
import subprocess

import numpy as np
import pytest

from chain_testlib import mutate, rand_seq, revcomp
from fasta_py import read_fastx

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
BIN = os.path.join(ROOT, "skani_b200", "skani-b200")
GOLD = os.path.join(ROOT, "tests", "golden")
EC, K12, VIR, O157 = (os.path.join(GOLD, f) for f in ("e.coli-EC590.fasta.gz", "e.coli-K12.fasta.gz", "viruses.fna", "o157_reads.fa.gz"))
FILES = [K12, VIR, EC]
HEADER = ["Ref_file", "Query_file", "Ref_contig", "Ref_start", "Ref_end", "Query_contig", "Query_start", "Query_end", "Strand",
          "Anchors", "Chunk_genome", "Chunk", "Chunk_ANI", "Chunk_weight"]
K, C = 15, 125


def run(args, env=None, ok=True):
    e = dict(os.environ)
    e.pop("SK_DEVICE_BUDGET_MB", None)
    e.update(env or {})
    p = subprocess.run([BIN] + args, capture_output=True, text=True, timeout=900, env=e)
    if ok:
        assert p.returncode == 0, p.stderr
    return p


def read_maps(path):
    lines = open(path).read().split("\n")
    assert lines[0].split("\t") == HEADER and lines[-1] == ""
    return [ln.split("\t") for ln in lines[1:-1]]


def contig_lengths(files):
    out = {}
    for f in files:
        for name, seq in read_fastx(f):
            out[(f, name)] = len(seq)
    return out


def check_against_rows(out, maps, ri=False, qi=False):
    """the distinct consecutive pairs of the mapping file are the printed rows, in order.  With -i style inputs a genome is a
    contig, named by the row's Ref_name / Query_name"""
    rows = [ln.split("\t") for ln in out.strip().split("\n")[1:]]
    key = lambda r: (r[0], r[1], r[5] if ri else "", r[6] if qi else "")
    mkey = lambda m: (m[0], m[1], m[2] if ri else "", m[5] if qi else "")
    seq = []
    for m in maps:
        if not seq or seq[-1] != mkey(m):
            seq.append(mkey(m))
    assert seq == [key(r) for r in rows]
    assert len(rows) > 0


def check_coords(maps, lengths):
    for m in maps:
        rs, re_, qs, qe = int(m[3]), int(m[4]), int(m[6]), int(m[7])
        assert 0 <= rs < re_ <= lengths[(m[0], m[2])], m
        assert 0 <= qs < qe <= lengths[(m[1], m[5])], m
        assert m[8] in "+-" and m[10] in "QR" and int(m[9]) >= 3
        assert m[12] == "NA" or 0 < float(m[12]) <= 100


@pytest.mark.parametrize("args,indiv", [
    (["dist", EC] + FILES, (False, False)),
    (["dist", EC] + FILES + ["-n", "1"], (False, False)),
    (["dist", "-q", O157, "--qi", "-r"] + FILES, (False, True)),
    (["dist", "-q", VIR, "-r", VIR, "--qi", "--ri", "--no-learned-ani"], (True, True)),
    (["triangle", "-E"] + FILES, (False, False)),
    (["triangle", "-E", "-i", VIR], (True, True)),
    (["triangle", "--detailed"] + FILES, None),
])
def test_main_output_unchanged(tmp_path, args, indiv):
    plain = run(args + ["-o", str(tmp_path / "a.tsv")])
    mp = str(tmp_path / "m.tsv")
    withm = run(args + ["-o", str(tmp_path / "b.tsv"), "--mappings", mp])
    assert open(tmp_path / "a.tsv").read() == open(tmp_path / "b.tsv").read()
    assert run(args).stdout == run(args + ["--mappings", str(tmp_path / "m2.tsv")]).stdout
    maps = read_maps(mp)
    assert open(mp).read() == open(tmp_path / "m2.tsv").read()
    check_coords(maps, contig_lengths(FILES + [O157]))
    if indiv is None:      # matrix output: the pairs are those of -E
        sparse = run([a for a in args if a != "--detailed"] + ["-E"]).stdout
        check_against_rows(sparse, maps)
    else:
        check_against_rows(open(tmp_path / "a.tsv").read(), maps, *indiv)
    del plain, withm


def test_fasta_equals_database_and_gpus_and_blocks(tmp_path):
    db = str(tmp_path / "db")
    run(["sketch"] + FILES + ["-o", db])
    base = ["dist", "-q", O157, "--qi", "-r"]
    ref = str(tmp_path / "fasta.tsv")
    run(base + FILES + ["--mappings", ref])
    outs = {}
    for name, args, env in [("db", base + [db], None), ("gpus2", base + FILES + ["--gpus", "2"], None),
                            ("blocks", base + FILES, {"SK_INTERMEDIATE_WRITE_COUNT": "37"})]:
        p = str(tmp_path / (name + ".tsv"))
        outs[name] = (run(args + ["--mappings", p], env).stdout, open(p).read())
    text = open(ref).read()
    assert len(text.split("\n")) > 300
    for name in ("db", "gpus2"):
        assert outs[name][1] == text, name
    # blocks of 37 queries: the main output groups rows block by block, and the mappings follow it row for row
    out37, text37 = outs["blocks"]
    assert sorted(text37.split("\n")) == sorted(text.split("\n"))
    check_against_rows(out37, read_maps(str(tmp_path / "blocks.tsv")), qi=True)
    # search against the same database: its printed pairs (ANI > 50) with their mappings
    p = str(tmp_path / "search.tsv")
    out = run(["search", "-d", db, EC, K12, "--mappings", p]).stdout
    assert out == run(["search", "-d", db, EC, K12]).stdout
    check_against_rows(out, read_maps(p))
    assert len(read_maps(p)) > 100


def test_planted_segments(tmp_path):
    """a 60 kb segment of the reference planted into an unrelated query forward at 20 kb and reverse-complemented at 150 kb"""
    rng = np.random.default_rng(5)
    L, seg = 300_000, 60_000
    ref = rand_seq(rng, L)
    q = rand_seq(rng, L)
    q[20_000:20_000 + seg] = mutate(rng, ref[50_000:50_000 + seg], 0.02)
    q[150_000:150_000 + seg] = mutate(rng, revcomp(ref[200_000:200_000 + seg]), 0.02)
    rf, qf = str(tmp_path / "ref.fa"), str(tmp_path / "query.fa")
    for path, name, s in [(rf, "ref_ctg", ref), (qf, "query_ctg", q)]:
        with open(path, "wb") as f:
            f.write(b">" + name.encode() + b"\n" + s.tobytes() + b"\n")
    mp = str(tmp_path / "m.tsv")
    run(["dist", qf, rf, "--mappings", mp, "--min-af", "0"])
    maps = read_maps(mp)
    assert maps and all(m[0] == rf and m[1] == qf and m[2] == "ref_ctg" and m[5] == "query_ctg" for m in maps)
    slack = K + C
    boxes = {"+": ((20_000, 80_000), (50_000, 110_000)), "-": ((150_000, 210_000), (200_000, 260_000))}
    covered = {"+": np.zeros(L, bool), "-": np.zeros(L, bool)}
    for m in maps:
        (qa, qb), (ra, rb) = boxes[m[8]]
        qs, qe, rs, re_ = int(m[6]), int(m[7]), int(m[3]), int(m[4])
        assert qa - slack <= qs < qe <= qb + slack and ra - slack <= rs < re_ <= rb + slack, m
        covered[m[8]][qs:qe] = True
    for s, ((qa, qb), _) in boxes.items():
        assert covered[s][qa:qb].mean() > 0.8, (s, covered[s][qa:qb].mean())


def test_refusals(tmp_path):
    mp = str(tmp_path / "m.tsv")
    for args, env, what in [(["dist", EC, K12], {"SK_DEVICE_BUDGET_MB": "8"}, "host sketch store"),
                            (["triangle", EC, K12], {"SK_DEVICE_BUDGET_MB": "8"}, "host sketch store"),
                            (["triangle", EC, K12, "--gpus", "2"], None, "--gpus")]:
        p = run(args + ["--mappings", mp], env, ok=False)
        assert p.returncode != 0 and p.stderr.startswith("ERROR") and what in p.stderr, (args, p.stderr)
    for cmd in ("cluster", "tree", "dereplicate", "sketch"):
        p = run([cmd, EC, K12, "--mappings", mp], ok=False)
        assert p.returncode == 2 and "--mappings" in p.stderr, (cmd, p.stderr)
