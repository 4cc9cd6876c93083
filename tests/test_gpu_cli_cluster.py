"""`skani-b200 cluster`: the cluster TSV equals the Python references (tests/cluster_ref.py) applied to the rows `triangle -E`
prints for the same inputs and flags, at thresholds midway between printed ANIs; it is byte-identical in memory, with
--gpus 2, on the store path, from a sketch database and from .sketch files; triangle-only flags and bad thresholds are refused."""
import os
import subprocess

import numpy as np
import pytest

import cluster_ref as R
from fasta_py import read_fastx

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
BIN = os.path.join(ROOT, "skani_b200", "skani-b200")
GOLD = os.path.join(ROOT, "tests", "golden")
EC, K12, VIR, TEST = (os.path.join(GOLD, f) for f in ("e.coli-EC590.fasta.gz", "e.coli-K12.fasta.gz", "viruses.fna", "test.fasta"))
HEADER = "Genome_file\tRepresentative_file\tCluster\tANI\tAlign_fraction_genome\tAlign_fraction_representative\tGenome_name\tRepresentative_name"


def run(args, env_add=None, rc=0):
    env = dict(os.environ)
    env.pop("SK_DEVICE_BUDGET_MB", None)
    env.update(env_add or {})
    p = subprocess.run([BIN] + args, capture_output=True, text=True, timeout=900, env=env)
    assert p.returncode == rc, p.stderr
    return p.stdout, p.stderr


@pytest.fixture(scope="module")
def synth_files(tmp_path_factory):
    """24 synthetic 150 kbp genomes in families, one FASTA file each"""
    from bench_support import synth
    d = tmp_path_factory.mktemp("synth")
    n, L = 24, 150_000
    bases, off, goc = synth.generate(0, n, L, G=6)
    files = []
    for g in range(n):
        path = str(d / ("g%02d.fa" % g))
        with open(path, "wb") as f:
            for i in np.nonzero(goc == g)[0]:
                f.write(b">g%02d_c%d synthetic\n" % (g, i) + bases[int(off[i]):int(off[i + 1])].tobytes() + b"\n")
        files.append(path)
    return files


def genomes(files, individual):
    """(file, first contig name, total length) per genome in genome-index order: (file name, record order), records >= 500 bp"""
    out = []
    for f in sorted(files):
        recs = [(name, len(seq)) for name, seq in read_fastx(f) if len(seq) >= 500]
        if individual:
            out += [(f, name, ln) for name, ln in recs]
        elif recs:
            out.append((f, recs[0][0], sum(ln for _, ln in recs)))
    return out


def expected(gen, tri_rows, t, single):
    """per genome: the set of rows the cluster output may print (several only where printed ANIs tie between representatives)"""
    n = len(gen)
    index = {(f, name): i for i, (f, name, _) in enumerate(gen)}
    a = np.array([index[(r[0], r[5])] for r in tri_rows], np.int64)
    b = np.array([index[(r[1], r[6])] for r in tri_rows], np.int64)
    ani = np.array([float(r[2]) / 100 for r in tri_rows], np.float32)
    total = np.array([ln for _, _, ln in gen], np.int64)
    order = np.lexsort((np.arange(n), -total))
    rank = np.empty(n, np.int64); rank[order] = np.arange(n)
    rep, cl, edge = R.reference(n, a, b, ani, np.float32(t / 100), rank, single)
    is_rep = rep == np.arange(n)
    lines = []
    for g in range(n):
        f, name, _ = gen[g]
        def line(rg, cols):
            return "\t".join([f, gen[rg][0], str(cl[g])] + cols + [name, gen[rg][1]])
        if is_rep[g]:
            lines.append({line(g, ["100.00"] * 3)})
            continue
        if edge[g] == R.NO_EDGE:
            lines.append({line(rep[g], ["NA"] * 3)})
            continue
        cand = [int(edge[g])]
        if not single:        # other representatives at the same printed ANI (the library compares the unrounded floats)
            best = float(tri_rows[cand[0]][2])
            cand = [i for i in range(len(tri_rows)) if g in (a[i], b[i]) and is_rep[a[i] + b[i] - g] and float(tri_rows[i][2]) == best]
        opts = set()
        for i in cand:
            r = tri_rows[i]
            afg, afr = (r[3], r[4]) if a[i] == g else (r[4], r[3])
            other = int(a[i] + b[i] - g)
            opts.add("\t".join([f, gen[other][0], str(cl[g]), r[2], afg, afr, name, gen[other][1]]))
        lines.append(opts)
    return lines, int(is_rep.sum())


def thresholds(tri_rows, k=4):
    printed = sorted({float(r[2]) for r in tri_rows if float(r[2]) > 10})
    mids = [(x + y) / 2 for x, y in zip(printed, printed[1:])]
    pick = [mids[int(i * (len(mids) - 1) / max(k - 1, 1))] for i in range(k)] if mids else []
    if printed:      # every row an edge / none: a printed value stands for the floats within 0.005 of it
        pick += [printed[0] - 0.006, min(printed[-1] + 0.006, 100.0)]
    return sorted({round(x, 4) for x in pick if 10 < x <= 100})


def check_against_triangle(inputs, flags, extra_t=()):
    individual = "-i" in flags
    tri, _ = run(["triangle", "-E"] + flags + inputs)
    rows = [ln.split("\t") for ln in tri.strip().split("\n")[1:] if ln]
    gen = genomes([x for x in inputs], individual)
    ts = thresholds(rows) + list(extra_t)
    assert ts
    counts = {}
    for t in ts:
        for single in (False, True):
            out, err = run(["cluster", "--ani", repr(t)] + (["--single-linkage"] if single else []) + flags + inputs)
            got = out.rstrip("\n").split("\n")
            assert got[0] == HEADER
            exp, n_clusters = expected(gen, rows, t, single)
            assert len(got) - 1 == len(exp) == len(gen)
            for g, (ln, opts) in enumerate(zip(got[1:], exp)):
                assert ln in opts, (t, single, g, ln, sorted(opts))
            assert "INFO %d genomes in %d clusters at ANI >= %s (%s)" % (len(gen), n_clusters, "%g" % t,
                                                                          "single linkage" if single else "greedy") in err
            counts[(t, single)] = n_clusters
    return counts


@pytest.mark.gpu
def test_ecoli_pair_one_and_two_clusters():
    counts = check_against_triangle([EC, K12], [], extra_t=(95.0, 99.0))
    tri, _ = run(["triangle", "-E", EC, K12])
    ani = float(tri.strip().split("\n")[1].split("\t")[2])
    assert 95.01 < ani and abs(ani - 99.0) > 0.01
    assert counts[(95.0, False)] == 1 and counts[(95.0, True)] == 1
    assert counts[(99.0, False)] == counts[(99.0, True)] == (1 if ani > 99.0 else 2)


@pytest.mark.gpu
@pytest.mark.parametrize("flags", [[], ["--min-af", "30"], ["--fast"]])
def test_goldens_match_triangle_rows(flags):
    check_against_triangle([EC, K12, VIR, TEST], flags)


@pytest.mark.gpu
def test_individual_records():
    check_against_triangle([VIR], ["-i"])


@pytest.mark.gpu
def test_synthetic_families_match_triangle_rows(synth_files):
    check_against_triangle(synth_files, [])


@pytest.mark.gpu
@pytest.mark.parametrize("single", [False, True])
def test_identical_on_every_path(synth_files, tmp_path, single):
    inputs = synth_files + [EC, K12, VIR]
    args = ["--ani", "97.5"] + (["--single-linkage"] if single else [])
    base, _ = run(["cluster"] + args + inputs)
    assert base.count("\n") == len(inputs) + 1
    assert single or "\tNA\t" not in base
    multi, err = run(["cluster", "--gpus", "2"] + args + inputs)
    assert multi == base
    store, err = run(["cluster"] + args + inputs, {"SK_DEVICE_BUDGET_MB": "8"})
    assert "Store path" in err and store == base
    db = str(tmp_path / "db")
    run(["sketch"] + inputs + ["-o", db])
    from_db, _ = run(["cluster"] + args + [db])
    assert from_db == base
    from_db_store, err = run(["cluster"] + args + [db], {"SK_DEVICE_BUDGET_MB": "8"})
    assert "Store path" in err and from_db_store == base
    sep = str(tmp_path / "sep")
    run(["sketch"] + inputs + ["-o", sep, "--separate-sketches"])
    sketches = sorted(os.path.join(sep, f) for f in os.listdir(sep) if f.endswith(".sketch"))
    assert len(sketches) == len(inputs)
    from_files, _ = run(["cluster"] + args + sketches)
    assert from_files == base
    out = str(tmp_path / "out.tsv")
    run(["cluster", "-o", out] + args + inputs)
    assert open(out).read() == base


@pytest.mark.parametrize("flag", [["-E"], ["--sparse"], ["--full-matrix"], ["--diagonal"], ["--distance"], ["--ci"], ["--detailed"],
                                  ["--ani", "10"], ["--ani", "100.5"], ["--ani", "-3"], ["--ani", "x"], ["--ani", "nan"]])
def test_refused_flags(flag):
    if not os.path.exists(BIN):
        import __graft_entry__ as g
        g.build()
    _, err = run(["cluster"] + flag + [VIR], rc=2)
    assert err.startswith("ERROR")
