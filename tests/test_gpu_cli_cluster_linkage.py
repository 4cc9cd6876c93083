"""`skani-b200 cluster --linkage average|complete [--dendrogram FILE]`: the cluster TSV equals the round procedure of
tests/linkage_ref.py applied to the rows `triangle -E` prints for the same inputs and flags, at cuts where that reference
gives the same answer with every printed ANI moved down or up by 0.005 % (so the 2-decimal printing cannot decide it); the
dendrogram file is a valid scipy linkage matrix whose fcluster at 100 - T is the TSV's partition; TSV and dendrogram are
byte-identical in memory, with --gpus 2, on the store path, from a sketch database and from .sketch files; the flag
refusals exit 2."""
import os

import numpy as np
import pytest

import linkage_ref as L
from test_gpu_cli_cluster import EC, HEADER, K12, TEST, VIR, genomes, run
from test_gpu_cli_cluster import synth_files  # noqa: F401  (fixture)


def reference(gen, rows, t, method, shift=0.0):
    n = len(gen)
    index = {(f, name): i for i, (f, name, _) in enumerate(gen)}
    a = np.array([index[(r[0], r[5])] for r in rows], np.int64)
    b = np.array([index[(r[1], r[6])] for r in rows], np.int64)
    ani = np.array([(float(r[2]) + shift) / 100 for r in rows], np.float32)
    total = np.array([ln for _, _, ln in gen], np.int64)
    order = np.lexsort((np.arange(n), -total))
    rank = np.empty(n, np.int64); rank[order] = np.arange(n)
    rep, cl, edge, _, _ = L.rounds(n, a, b, ani, rank, method, float(np.float32(t / 100)), False)
    return rep, cl, edge


def stable_cuts(gen, rows, method, k=4):
    """cuts midway between printed ANIs (plus 95 and 99) at which the answer does not move with the printing's rounding"""
    printed = sorted({float(r[2]) for r in rows if float(r[2]) > 10})
    mids = [(x + y) / 2 for x, y in zip(printed, printed[1:])]
    cand = sorted({round(x, 4) for x in mids + [95.0, 99.0] if 10 < x <= 100})
    out = []
    for t in cand:
        base = reference(gen, rows, t, method)
        if all(all(np.array_equal(x, y) for x, y in zip(base, reference(gen, rows, t, method, s))) for s in (-0.005, 0.005)):
            out.append(t)
    return [out[int(i * (len(out) - 1) / max(k - 1, 1))] for i in range(min(k, len(out)))]


def check_against_triangle(inputs, flags, tmp_path):
    from scipy.cluster.hierarchy import fcluster, is_valid_linkage
    tri, _ = run(["triangle", "-E"] + flags + inputs)
    rows = [ln.split("\t") for ln in tri.strip().split("\n")[1:] if ln]
    gen = genomes(inputs, "-i" in flags)
    by_pair = {}
    index = {(f, name): i for i, (f, name, _) in enumerate(gen)}
    for r in rows:
        x, y = index[(r[0], r[5])], index[(r[1], r[6])]
        by_pair[(x, y)] = (r, False)
        by_pair[(y, x)] = (r, True)
    checked = 0
    for method in L.METHODS:
        cuts = stable_cuts(gen, rows, method)
        assert cuts
        for t in cuts:
            z = str(tmp_path / "z.tsv")
            out, err = run(["cluster", "--ani", repr(t), "--linkage", method, "--dendrogram", z] + flags + inputs)
            got = out.rstrip("\n").split("\n")
            assert got[0] == HEADER and len(got) - 1 == len(gen)
            rep, cl, edge = reference(gen, rows, t, method)
            for g, ln in enumerate(got[1:]):
                f, name, _ = gen[g]
                r = int(rep[g])
                if r == g:
                    cols = ["100.00"] * 3
                elif edge[g] == L.NO_EDGE:
                    cols = ["NA"] * 3
                else:
                    row, flipped = by_pair[(g, r)]
                    cols = [row[2], row[4], row[3]] if flipped else [row[2], row[3], row[4]]
                assert ln == "\t".join([f, gen[r][0], str(cl[g])] + cols + [name, gen[r][1]]), (method, t, g)
            n_clusters = int(cl.max()) + 1
            assert "INFO %d genomes in %d clusters at ANI >= %s (%s linkage, " % (len(gen), n_clusters, "%g" % t, method) in err
            Z = np.loadtxt(z, ndmin=2)
            assert Z.shape == (len(gen) - 1, 4) and is_valid_linkage(Z)
            if np.min(np.abs(Z[:, 2] - (100 - t))) > 1e-5:
                tsv_cl = [int(ln.split("\t")[2]) for ln in got[1:]]
                assert L.partition(fcluster(Z, 100 - t, "distance")) == L.partition(tsv_cl), (method, t)
            checked += 1
    return checked


@pytest.mark.gpu
@pytest.mark.parametrize("flags", [[], ["--min-af", "30"]])
def test_goldens_match_triangle_rows(flags, tmp_path):
    assert check_against_triangle([EC, K12, VIR, TEST], flags, tmp_path)


@pytest.mark.gpu
def test_individual_records(tmp_path):
    assert check_against_triangle([VIR], ["-i"], tmp_path)


@pytest.mark.gpu
def test_synthetic_families_match_triangle_rows(synth_files, tmp_path):  # noqa: F811
    assert check_against_triangle(synth_files, [], tmp_path)


@pytest.mark.gpu
@pytest.mark.parametrize("method", L.METHODS)
def test_identical_on_every_path(synth_files, tmp_path, method):  # noqa: F811
    inputs = synth_files + [EC, K12, VIR]
    z = str(tmp_path / "z.tsv")

    def both(extra, env=None):
        out, err = run(["cluster", "--ani", "97.5", "--linkage", method, "--dendrogram", z] + extra, env)
        return out, open(z).read(), err
    base, zbase, _ = both(inputs)
    assert base.count("\n") == len(inputs) + 1 and zbase.count("\n") == len(inputs) - 1
    assert both(["--gpus", "2"] + inputs)[:2] == (base, zbase)
    store = both(inputs, {"SK_DEVICE_BUDGET_MB": "8"})
    assert "Store path" in store[2] and store[:2] == (base, zbase)
    db = str(tmp_path / "db")
    run(["sketch"] + inputs + ["-o", db])
    assert both([db])[:2] == (base, zbase)
    sep = str(tmp_path / "sep")
    run(["sketch"] + inputs + ["-o", sep, "--separate-sketches"])
    sketches = sorted(os.path.join(sep, f) for f in os.listdir(sep) if f.endswith(".sketch"))
    assert len(sketches) == len(inputs)
    assert both(sketches)[:2] == (base, zbase)
    # without --dendrogram the TSV is the same
    out, _ = run(["cluster", "--ani", "97.5", "--linkage", method] + inputs)
    assert out == base


@pytest.mark.parametrize("flag", [["--linkage", "single"], ["--linkage", "ward"], ["--linkage", "average", "--single-linkage"],
                                  ["--single-linkage", "--linkage", "complete"], ["--dendrogram", "z.tsv"],
                                  ["--single-linkage", "--dendrogram", "z.tsv"], ["--linkage", "average", "-E"]])
def test_refused_flags(flag, tmp_path):
    from test_gpu_cli_cluster import BIN
    if not os.path.exists(BIN):
        import __graft_entry__ as g
        g.build()
    flag = [str(tmp_path / x) if x.endswith(".tsv") else x for x in flag]
    _, err = run(["cluster"] + flag + [VIR], rc=2)
    assert err.startswith("ERROR")
    assert not os.path.exists(str(tmp_path / "z.tsv"))
