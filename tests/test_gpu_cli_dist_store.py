"""`skani-b200 dist` on the store path (references and queries kept in host sketch stores, chained in working sets; forced
here with a small SK_DEVICE_BUDGET_MB): stdout and the "INFO Writing results" lines must equal the default in-memory run byte
for byte, for FASTA and .sketch inputs on either side, --qi / --ri, reads in intermediate-write blocks with -n, --ci and
--detailed, and --gpus 3; stderr must name the store path."""
import os
import subprocess

import pytest

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
BIN = os.path.join(ROOT, "skani_b200", "skani-b200")
GOLD = os.path.join(ROOT, "tests", "golden")
EC, K12, VIR, O157 = (os.path.join(GOLD, f) for f in ("e.coli-EC590.fasta.gz", "e.coli-K12.fasta.gz", "viruses.fna", "o157_reads.fa.gz"))
FILES = [K12, VIR, EC]
BUDGET_MB = "8"      # about 2 MB per E. coli sketch: a few working sets


def run(args, budget=None, write_count=None, out=None):
    env = dict(os.environ)
    env.pop("SK_DEVICE_BUDGET_MB", None)
    if budget:
        env["SK_DEVICE_BUDGET_MB"] = budget
    if write_count:
        env["SK_INTERMEDIATE_WRITE_COUNT"] = str(write_count)
    p = subprocess.run([BIN] + args + (["-o", out] if out else []), capture_output=True, text=True, timeout=900, env=env)
    assert p.returncode == 0, p.stderr
    text = open(out).read() if out else p.stdout
    return text, [ln for ln in p.stderr.splitlines() if ln.startswith("INFO Writing results")], p.stderr


def same_on_store_path(args, write_count=None, min_rows=1, tmp_path=None):
    outs = [None, None] if tmp_path is None else [str(tmp_path / "mem.tsv"), str(tmp_path / "store.tsv")]
    mem = run(args, None, write_count, outs[0])
    store = run(args, BUDGET_MB, write_count, outs[1])
    assert "INFO Store path" in store[2] and "INFO Store path" not in mem[2]
    assert store[:2] == mem[:2]
    assert len(mem[0].strip().split("\n")) - 1 >= min_rows
    return mem


def test_dist_fasta(tmp_path):
    same_on_store_path(["dist", EC] + FILES, min_rows=2)
    same_on_store_path(["dist", EC] + FILES, min_rows=2, tmp_path=tmp_path)          # -o
    same_on_store_path(["dist", "-q", VIR, "-r", VIR, "--qi", "--ri"], min_rows=3)


@pytest.mark.parametrize("flags", [[], ["-n", "2"], ["--ci"], ["--detailed"]])
def test_dist_reads_in_blocks(flags):
    _, flushes, _ = same_on_store_path(["dist", "-q", O157, "--qi", "-r"] + FILES + flags, write_count=37, min_rows=200)
    assert len(flushes) >= 5                                                  # blocks of 37 reads


@pytest.fixture(scope="module")
def sketches(tmp_path_factory):
    sep = str(tmp_path_factory.mktemp("sk") / "sep")
    run(["sketch"] + FILES + ["-o", sep, "--separate-sketches"])
    return sep, [os.path.join(sep, os.path.basename(f) + ".sketch") for f in FILES]


def test_dist_sketch_files(sketches):
    sep, sk_files = sketches
    _, _, err = same_on_store_path(["dist", "-q", O157, "--qi", "-r"] + sk_files + [os.path.join(sep, "markers.bin")], write_count=37, min_rows=200)
    assert "INFO Sketches detected" in err
    same_on_store_path(["dist", "-q"] + sk_files + ["-r"] + sk_files, min_rows=3)
    same_on_store_path(["dist", "-q"] + sk_files + ["-r"] + FILES, min_rows=3)


def test_dist_gpus_3():
    same_on_store_path(["dist", "-q", O157, "--qi", "-r"] + FILES + ["--gpus", "3"], write_count=37, min_rows=200)
    same_on_store_path(["dist", EC] + FILES + ["--gpus", "3"], min_rows=2)
