"""`skani-b200 dereplicate`: stdout and -o byte-identical to `cluster`'s greedy TSV on FASTA inputs, .sketch files and a
sketch database, with one genome per wave (SK_DEREP_WAVE=1) and the default waves, with and without -i and --faster-small;
--representatives lists the TSV's representatives in cluster order; every refusal is an ERROR line and a non-zero exit."""
import os
import subprocess

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
BIN = os.path.join(ROOT, "skani_b200", "skani-b200")
GOLD = os.path.join(ROOT, "tests", "golden")
EC, K12, VIR, TEST = (os.path.join(GOLD, f) for f in ("e.coli-EC590.fasta.gz", "e.coli-K12.fasta.gz", "viruses.fna", "test.fasta"))


def run(args, env_add=None, rc=0):
    env = dict(os.environ)
    for k in ("SK_DEVICE_BUDGET_MB", "SK_DEREP_WAVE"):
        env.pop(k, None)
    env.update(env_add or {})
    p = subprocess.run([BIN] + args, capture_output=True, text=True, timeout=900, env=env)
    assert p.returncode == rc, p.stderr
    return p.stdout, p.stderr


@pytest.fixture(scope="module")
def synth_files(tmp_path_factory):
    """40 synthetic 120 kbp genomes in families of 8, one FASTA file each"""
    from bench_support import synth
    d = tmp_path_factory.mktemp("synth")
    n, L = 40, 120_000
    bases, off, goc = synth.generate(0, n, L, G=8)
    files = []
    for g in range(n):
        path = str(d / ("g%02d.fa" % g))
        with open(path, "wb") as f:
            for i in np.nonzero(goc == g)[0]:
                f.write(b">g%02d_c%d synthetic\n" % (g, i) + bases[int(off[i]):int(off[i + 1])].tobytes() + b"\n")
        files.append(path)
    return files


def same_as_cluster(inputs, flags, tmp_path):
    """dereplicate == cluster byte for byte, at every wave setting; returns the TSV"""
    base, _ = run(["cluster"] + flags + inputs)
    reps = str(tmp_path / "reps.txt")
    for env in ({"SK_DEREP_WAVE": "1"}, {"SK_DEREP_WAVE": "3"}, {}):
        out, err = run(["dereplicate", "--representatives", reps] + flags + inputs, env)
        assert out == base, (env, flags)
        assert "INFO %d genomes in " % (base.count("\n") - 1) in err and "pairs screened" in err
        rows = [ln.split("\t") for ln in base.rstrip("\n").split("\n")[1:]]
        individual = "-i" in flags
        want = {}
        for r in rows:
            if r[0] == r[1] and (not individual or r[6] == r[7]):
                want[int(r[2])] = r[6] if individual else r[0]
        assert open(reps).read().split("\n")[:-1] == [want[c] for c in range(len(want))]
    o = str(tmp_path / "out.tsv")
    run(["dereplicate", "-o", o] + flags + inputs)
    assert open(o).read() == base
    return base


@pytest.mark.gpu
@pytest.mark.parametrize("ani", ["80", "95", "99"])
def test_fasta_inputs(synth_files, tmp_path, ani):
    base = same_as_cluster(synth_files + [EC, K12, VIR, TEST], ["--ani", ani], tmp_path)
    assert base.count("\n") >= len(synth_files) + 4


@pytest.mark.gpu
@pytest.mark.parametrize("flags", [["-i"], ["-i", "--faster-small"], ["--faster-small"], ["--min-af", "40"]])
def test_flags(tmp_path, flags):
    same_as_cluster([VIR, EC, K12], flags, tmp_path)


@pytest.mark.gpu
def test_sketch_inputs(synth_files, tmp_path):
    inputs = synth_files + [EC, K12, VIR]
    base, _ = run(["cluster", "--ani", "97.5"] + inputs)
    db = str(tmp_path / "db")
    run(["sketch"] + inputs + ["-o", db])
    assert same_as_cluster([db], ["--ani", "97.5"], tmp_path) == base
    sep = str(tmp_path / "sep")
    run(["sketch"] + inputs + ["-o", sep, "--separate-sketches"])
    sketches = sorted(os.path.join(sep, f) for f in os.listdir(sep) if f.endswith(".sketch"))
    assert same_as_cluster(sketches, ["--ani", "97.5"], tmp_path) == base


@pytest.mark.gpu
def test_store_path_refused(synth_files):
    _, err = run(["dereplicate"] + synth_files, {"SK_DEVICE_BUDGET_MB": "8"}, rc=1)
    assert err.startswith("ERROR") and "use cluster" in err


@pytest.mark.parametrize("flag", [["--single-linkage"], ["--linkage", "average"], ["--dendrogram", "z.tsv"], ["-E"], ["--sparse"],
                                  ["--full-matrix"], ["--diagonal"], ["--distance"], ["--ci"], ["--detailed"], ["--gpus", "2"],
                                  ["--ani", "10"], ["--ani", "x"]])
def test_refused_flags(flag):
    if not os.path.exists(BIN):
        import __graft_entry__ as g
        g.build()
    _, err = run(["dereplicate"] + flag + [VIR], rc=2)
    assert err.startswith("ERROR")
    if flag[0] in ("--single-linkage", "--linkage", "--dendrogram", "--gpus"):
        assert "cluster" in err
