"""`skani-b200 dereplicate --host-store`: stdout, -o and --representatives byte-identical to in-memory `dereplicate` and
stdout to `cluster`'s greedy TSV, with SK_DEVICE_BUDGET_MB unset and small, --gpus 1 and 2 (contexts share GPU 0 when only one
device is visible) and SK_DEREP_WAVE 1 and unset; on FASTA inputs (40 synthetic genomes plus the goldens), a sketch database,
.sketch files, -i, --faster-small and --min-af 40.  --host-store is a dereplicate option only."""
import os
import subprocess

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
BIN = os.path.join(ROOT, "skani_b200", "skani-b200")
GOLD = os.path.join(ROOT, "tests", "golden")
EC, K12, VIR, TEST = (os.path.join(GOLD, f) for f in ("e.coli-EC590.fasta.gz", "e.coli-K12.fasta.gz", "viruses.fna", "test.fasta"))
BUDGET_MB = "8"      # about 2 MB per E. coli sketch: many working sets, none over budget / 2
SETTINGS = [         # (SK_DEVICE_BUDGET_MB, --gpus, SK_DEREP_WAVE)
    (None, "1", None),
    (BUDGET_MB, "1", "1"),
    (BUDGET_MB, "2", None),
    (None, "2", "1"),
]


def run(args, env_add=None, rc=0):
    env = dict(os.environ)
    for k in ("SK_DEVICE_BUDGET_MB", "SK_DEREP_WAVE", "SK_TRACE"):
        env.pop(k, None)
    env.update({k: v for k, v in (env_add or {}).items() if v is not None})
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


def outputs(cmd, inputs, flags, tmp_path, env=None):
    """(stdout, -o file, --representatives file, stderr) of one dereplicate run"""
    o, reps = str(tmp_path / "out.tsv"), str(tmp_path / "reps.txt")
    out, err = run(cmd + flags + inputs, env)
    run(cmd + ["-o", o, "--representatives", reps] + flags + inputs, env)
    return out, open(o).read(), open(reps).read(), err


def same_on_host_store(inputs, flags, tmp_path, settings=SETTINGS):
    """dereplicate --host-store == in-memory dereplicate == cluster, in every setting; returns the TSV"""
    base, _ = run(["cluster"] + flags + inputs)
    mem = outputs(["dereplicate"], inputs, flags, tmp_path)
    assert mem[0] == base and mem[1] == base and "INFO Store path" not in mem[3]
    for budget, gpus, wave in settings:
        env = {"SK_DEVICE_BUDGET_MB": budget, "SK_DEREP_WAVE": wave}
        got = outputs(["dereplicate", "--host-store", "--gpus", gpus], inputs, flags, tmp_path, env)
        assert got[:3] == mem[:3], (budget, gpus, wave, flags)
        err = got[3]
        assert "INFO Store path:" in err and "pairs screened" in err and "working sets" in err, err
    return base


@pytest.mark.gpu
def test_fasta_inputs(synth_files, tmp_path):
    base = same_on_host_store(synth_files + [EC, K12, VIR, TEST], ["--ani", "95"], tmp_path)
    assert base.count("\n") >= len(synth_files) + 4


@pytest.mark.gpu
@pytest.mark.parametrize("flags", [["-i"], ["--faster-small"], ["--min-af", "40"]])
def test_flags(tmp_path, flags):
    same_on_host_store([VIR, EC, K12], flags, tmp_path, settings=SETTINGS[:3])


@pytest.mark.gpu
def test_sketch_inputs(synth_files, tmp_path):
    inputs = synth_files + [EC, K12, VIR]
    base, _ = run(["cluster", "--ani", "97.5"] + inputs)
    db = str(tmp_path / "db")
    run(["sketch"] + inputs + ["-o", db])
    assert same_on_host_store([db], ["--ani", "97.5"], tmp_path) == base
    sep = str(tmp_path / "sep")
    run(["sketch"] + inputs + ["-o", sep, "--separate-sketches"])
    sketches = sorted(os.path.join(sep, f) for f in os.listdir(sep) if f.endswith(".sketch"))
    assert same_on_host_store(sketches, ["--ani", "97.5"], tmp_path, settings=SETTINGS[1:3]) == base


@pytest.mark.parametrize("cmd", ["cluster", "triangle", "tree", "dist"])
def test_other_commands_refuse_the_flag(cmd):
    if not os.path.exists(BIN):
        import __graft_entry__ as g
        g.build()
    _, err = run([cmd, "--host-store", VIR, VIR], rc=2)
    assert err.startswith("ERROR unknown option --host-store")
