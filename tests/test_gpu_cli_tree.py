"""`skani-b200 tree [--method nj|average|complete]`: valid Newick with every genome's label exactly once; the NJ topology
equals tests/nj_ref.py applied to the rows `triangle -E` prints, wherever moving every printed ANI down or up by 0.005 %
leaves the reference's topology unchanged (so the 2-decimal printing cannot decide it); the average / complete trees'
patristic distances equal scipy's cophenetic distances of `cluster --linkage ... --dendrogram`'s matrix; the output is
byte-identical in memory, with --gpus 2, on the store path, from a sketch database and from .sketch files; labels with
spaces or quotes are quoted; the flag refusals exit 2."""
import os
import shutil

import numpy as np
import pytest

import nj_ref as N
from test_gpu_cli_cluster import BIN, EC, K12, TEST, VIR, genomes, run
from test_gpu_cli_cluster import synth_files  # noqa: F401  (fixture)


def triangle_rows(inputs, flags):
    tri, _ = run(["triangle", "-E"] + flags + inputs)
    rows = [ln.split("\t") for ln in tri.strip().split("\n")[1:] if ln]
    gen = genomes(inputs, "-i" in flags)
    index = {(f, name): i for i, (f, name, _) in enumerate(gen)}
    a = np.array([index[(r[0], r[5])] for r in rows], np.int64)
    b = np.array([index[(r[1], r[6])] for r in rows], np.int64)
    printed = np.array([float(r[2]) for r in rows])
    return gen, a, b, printed


def parse(text, names):
    labels, parent, length = N.parse_newick(text)
    assert sorted(labels) == sorted(names) and len(set(labels)) == len(labels)
    return labels, parent, length


def check_nj(inputs, flags):
    """True when the printed rows pin the reference's topology and the tree has it"""
    gen, a, b, printed = triangle_rows(inputs, flags)
    names = [g[1] if "-i" in flags else g[0] for g in gen]
    out, err = run(["tree"] + flags + inputs)
    assert out.endswith(";\n") and out.count("\n") == 1
    assert "INFO %d genomes, tree by nj (" % len(gen) in err
    labels, parent, _ = parse(out, names)
    if len(gen) < 4:
        return False

    def ref(shift):
        joins = N.nj_results(len(gen), a, b, ((printed + shift) / 100).astype(np.float32))
        return N.splits(len(gen), N.tree_of_joins(len(gen), joins)[0])
    want = ref(0.0)
    if any(ref(s) != want for s in (-0.005, 0.005)):
        return False
    assert N.newick_splits(labels, parent, names) == want
    return True


@pytest.mark.gpu
@pytest.mark.parametrize("flags", [[], ["--min-af", "30"]])
def test_goldens_nj(flags):
    check_nj([EC, K12, VIR, TEST], flags)


@pytest.mark.gpu
def test_individual_records():
    check_nj([VIR], ["-i"])


@pytest.mark.gpu
def test_synthetic_nj(synth_files):  # noqa: F811
    assert check_nj(synth_files, [])


@pytest.mark.gpu
@pytest.mark.parametrize("method", ["average", "complete"])
def test_linkage_patristic_is_cophenetic(synth_files, tmp_path, method):  # noqa: F811
    from scipy.cluster.hierarchy import cophenet
    from scipy.spatial.distance import squareform
    inputs = synth_files + [EC, K12, VIR]
    gen = genomes(inputs, False)
    names = [g[0] for g in gen]
    out, err = run(["tree", "--method", method] + inputs)
    assert "INFO %d genomes, tree by %s (" % (len(gen), method) in err
    labels, parent, length = parse(out, names)
    assert sum(p < 0 for p in parent) == 1 and all(len([c for c in parent if c == v]) in (0, 2) for v in range(len(parent)))
    P = N.patristic(len(labels), parent, length)
    order = [labels.index(x) for x in names]
    P = P[np.ix_(order, order)]
    z = str(tmp_path / "z.tsv")
    run(["cluster", "--linkage", method, "--dendrogram", z] + inputs)
    C = squareform(cophenet(np.loadtxt(z, ndmin=2)))
    assert np.allclose(P, C, rtol=0, atol=2e-5 * len(gen))


@pytest.mark.gpu
@pytest.mark.parametrize("method", ["nj", "average"])
def test_identical_on_every_path(synth_files, tmp_path, method):  # noqa: F811
    inputs = synth_files + [EC, K12, VIR]
    flags = ["--method", method]
    base, _ = run(["tree"] + flags + inputs)
    assert base.count("\n") == 1
    assert run(["tree", "--gpus", "2"] + flags + inputs)[0] == base
    store = run(["tree"] + flags + inputs, {"SK_DEVICE_BUDGET_MB": "8"})
    assert "Store path" in store[1] and store[0] == base
    db = str(tmp_path / "db")
    run(["sketch"] + inputs + ["-o", db])
    assert run(["tree"] + flags + [db])[0] == base
    sep = str(tmp_path / "sep")
    run(["sketch"] + inputs + ["-o", sep, "--separate-sketches"])
    sketches = sorted(os.path.join(sep, f) for f in os.listdir(sep) if f.endswith(".sketch"))
    assert len(sketches) == len(inputs)
    assert run(["tree"] + flags + sketches)[0] == base
    o = str(tmp_path / "t.nwk")
    run(["tree", "-o", o] + flags + inputs)
    assert open(o).read() == base


@pytest.mark.gpu
def test_labels_quoted(synth_files, tmp_path):  # noqa: F811
    d = tmp_path / "odd names"
    d.mkdir()
    files = []
    for k, name in enumerate(["plain.fa", "with space.fa", "it's.fa", "a,b(c):d;[e].fa"]):
        p = str(d / name)
        shutil.copy(synth_files[k], p)
        files.append(p)
    out, _ = run(["tree"] + files)
    for p in files:
        assert "'" + p.replace("'", "''") + "'" in out
    parse(out, files)


@pytest.mark.parametrize("flag", [["-E"], ["--sparse"], ["--full-matrix"], ["--diagonal"], ["--distance"], ["--ci"], ["--detailed"],
                                  ["--method", "upgma"], ["--ani", "95"], ["--linkage", "average"], ["--dendrogram", "z.tsv"],
                                  ["--single-linkage"]])
def test_refused_flags(flag, tmp_path):
    if not os.path.exists(BIN):
        import __graft_entry__ as g
        g.build()
    flag = [str(tmp_path / x) if x.endswith(".tsv") else x for x in flag]
    out, err = run(["tree"] + flag + [VIR], rc=2)
    assert err.startswith("ERROR") and out == ""
    assert not os.path.exists(str(tmp_path / "z.tsv"))
