"""`skani-b200 search` over query groups: every way of cutting the queries into groups (SK_SKETCH_GROUP_FILES, the bases bound
SK_SEARCH_GROUP_BASES cutting one --qi read file, write blocks that straddle groups, forced reference index parts) gives
byte-identical stdout, -o file, `INFO Writing results` lines and --mappings file to the run with one group, on consolidated
and --separate-sketches databases, with -n 1 and --gpus 2, for FASTA and .sketch queries; and a multi-group run equals the
oracle's search rows, including queries named like a reference and queries whose names sort between references."""
import os
import shutil
import subprocess

import numpy as np
import pytest

import oracle_py as O

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
BIN = os.path.join(ROOT, "skani_b200", "skani-b200")
GOLD = os.path.join(ROOT, "tests", "golden")
EC, K12, VIR, O157 = (os.path.join(GOLD, f) for f in ("e.coli-EC590.fasta.gz", "e.coli-K12.fasta.gz", "viruses.fna", "o157_reads.fa.gz"))
FILES = [K12, VIR, EC]


def run(args, env=None, tmp=None):
    """(stdout, INFO Writing results lines, -o file, --mappings file, number of query groups) of one search run; with tmp the
    run writes -o and --mappings there, otherwise --mappings only"""
    env = dict(os.environ, **(env or {}))
    extra = []
    out = maps = None
    if tmp is not None:
        out, maps = os.path.join(tmp, "out.tsv"), os.path.join(tmp, "maps.tsv")
        extra = ["-o", out, "--mappings", maps]
    p = subprocess.run([BIN] + args + extra, capture_output=True, text=True, timeout=900, env=env)
    assert p.returncode == 0, p.stderr
    groups = [ln for ln in p.stderr.splitlines() if ln.startswith("INFO Query group ")]
    flushes = [ln for ln in p.stderr.splitlines() if ln.startswith("INFO Writing results")]
    files = tuple(open(f).read() if f else None for f in (out, maps))
    return (p.stdout, flushes) + files, len(groups)


def same(args, envs, tmp_path, groups=None, common=None):
    """every env's run equals the run with one group (common: variables of every run); groups[i] = the expected group count of
    envs[i]"""
    common = common or {}
    base, n1 = run(args, common, tmp=str(tmp_path))
    base_stdout, _ = run(args, common)
    assert n1 == 1
    for i, env in enumerate(envs):
        env = dict(common, **env)
        got, n = run(args, env, tmp=str(tmp_path))
        assert got == base, env
        assert run(args, env)[0] == base_stdout, env
        if groups is not None:
            assert n == groups[i], (env, n)
    return base, base_stdout


@pytest.fixture(scope="module")
def dbs(tmp_path_factory):
    d = tmp_path_factory.mktemp("dbs")
    db, sep = str(d / "db"), str(d / "sep")
    run(["sketch"] + FILES + ["-o", db])
    run(["sketch"] + FILES + ["-o", sep, "--separate-sketches"])
    return db, sep


@pytest.mark.parametrize("layout", ["consolidated", "separate"])
def test_file_groups(dbs, layout, tmp_path):
    db = dbs[0] if layout == "consolidated" else dbs[1]
    envs = [{"SK_SKETCH_GROUP_FILES": "1"}, {"SK_SKETCH_GROUP_FILES": "2"},
            {"SK_SKETCH_GROUP_FILES": "1", "SK_REF_INDEX_PART_MARKERS": "3000"}]
    base, _ = same(["search", "-d", db] + FILES, envs, tmp_path, groups=[3, 2, 3])
    assert len(base[0].splitlines()) == 0 and base[2].count("\n") >= 4          # rows went to -o, header + 3 or more
    _, out = same(["search", "-d", db] + FILES, envs, tmp_path, groups=[3, 2, 3], common={"SK_INTERMEDIATE_WRITE_COUNT": "2"})
    assert len(out[1]) == 1                                                  # blocks of two queries: one flush line
    same(["search", "-d", db] + FILES + ["-n", "1", "--gpus", "2"], envs[:1], tmp_path, groups=[3])


@pytest.mark.parametrize("flags", [[], ["-n", "1"], ["--gpus", "2"]])
def test_reads_cut_into_groups(dbs, flags, tmp_path):
    # 364 reads (5.5 Mbp) in about four groups; blocks of 37 reads straddle them
    env = {"SK_SEARCH_GROUP_BASES": "1500000"}
    wc = {"SK_INTERMEDIATE_WRITE_COUNT": "37"}
    base, _ = same(["search", "-d", dbs[0], O157, "--qi"] + flags, [env, dict(env, SK_REF_INDEX_PART_MARKERS="2500")], tmp_path, common=wc)
    _, n = run(["search", "-d", dbs[0], O157, "--qi"] + flags, dict(env, **wc))
    assert n >= 4
    assert len(base[1]) == 364 // 37                                       # 10 blocks: 9 flush lines
    if not flags:
        assert base[2].count("\n") > 100 and base[3].count("\n") > 100


def test_sketch_queries_in_name_order(dbs, tmp_path):
    # .sketch copies whose path order is the reverse of the names stored in them
    sep = dbs[1]
    qdir = tmp_path / "q"
    qdir.mkdir()
    qs = []
    for f, p in zip(sorted(FILES), ("z.sketch", "y.sketch", "x.sketch")):
        shutil.copy(os.path.join(sep, os.path.basename(f) + ".sketch"), qdir / p)
        qs.append(str(qdir / p))
    base, _ = same(["search", "-d", dbs[0]] + qs, [{"SK_SKETCH_GROUP_FILES": "1"}, {"SK_SKETCH_GROUP_FILES": "2"}], tmp_path, groups=[3, 2])
    assert base[2].count("\n") >= 4                                        # header + 3 or more rows


def f2(x):
    return "%.2f" % float(np.float32(x) * np.float32(100.0))


def test_names_between_references_and_oracle(tmp_path):
    # references a_EC590, c_K12, e_viruses; queries named before all, equal to a reference, between two, and after all.  Equal
    # genomes under different names exercise the file-name tie-break of the chain.
    rdir = tmp_path / "r"
    rdir.mkdir()
    refs = [str(rdir / n) for n in ("a_EC590.fasta.gz", "c_K12.fasta.gz", "e_viruses.fna")]
    for src, dst in zip((EC, K12, VIR), refs):
        shutil.copy(src, dst)
    queries = [str(rdir / n) for n in ("0_K12.fasta.gz", "b_EC590.fasta.gz", "d_K12.fasta.gz", "z_EC590.fasta.gz")]
    for src, dst in zip((K12, EC, K12, EC), queries):
        shutil.copy(src, dst)
    queries.append(refs[1])
    db = str(tmp_path / "db")
    run(["sketch"] + refs + ["-o", db])
    base, _ = same(["search", "-d", db] + queries, [{"SK_SKETCH_GROUP_FILES": "1"}, {"SK_SKETCH_GROUP_FILES": "3"}], tmp_path, groups=[5, 2])
    got, _ = run(["search", "-d", db] + queries, {"SK_SKETCH_GROUP_FILES": "1"})
    osk, _ = O.sketch_files(refs)
    q, _ = O.sketch_files(queries)
    exp = O.search(osk, q, O.cmd(learned_ani=True, min_af=-1.0, rescue_small=False))
    want = sorted((osk[r.ref_id].file_name, q[r.query_id].file_name, f2(r.ani), f2(r.af_ref), f2(r.af_query),
                   osk[r.ref_id].contig_name(0), q[r.query_id].contig_name(0)) for r in exp)
    rows = sorted(tuple(ln.split("\t")[:7]) for ln in got[0].splitlines()[1:])
    assert rows == want and len(want) >= 2 * len(queries)
    assert any(r[0] == r[1] for r in rows)                                  # a query named like its reference
