"""`skani-b200 dist --gpus N` and `search --gpus N` split the references over N contexts (here all on GPU 0, which takes the
same path as N GPUs); stdout must be byte-identical to the run without the flag, intermediate flushes included."""
import os
import subprocess

import pytest

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
BIN = os.path.join(ROOT, "skani_b200", "skani-b200")
GOLD = os.path.join(ROOT, "tests", "golden")
EC, K12, VIR, O157 = (os.path.join(GOLD, f) for f in ("e.coli-EC590.fasta.gz", "e.coli-K12.fasta.gz", "viruses.fna", "o157_reads.fa.gz"))
FILES = [K12, VIR, EC]


def run(args, write_count=None, env=None):
    env = dict(os.environ, **(env or {}))
    if write_count:
        env["SK_INTERMEDIATE_WRITE_COUNT"] = str(write_count)
    p = subprocess.run([BIN] + args, capture_output=True, text=True, timeout=900, env=env)
    assert p.returncode == 0, p.stderr
    return p.stdout, [ln for ln in p.stderr.splitlines() if ln.startswith("INFO Writing results")]


def same_with_gpus(args, write_count=None, min_rows=1):
    one = run(args, write_count)
    three = run(args + ["--gpus", "3"], write_count)
    assert three == one
    assert len(one[0].strip().split("\n")) - 1 >= min_rows
    return one


def test_dist_fasta_refs():
    same_with_gpus(["dist", EC] + FILES, min_rows=2)                       # EC590 against K12, viruses, EC590
    same_with_gpus(["dist", "-q", VIR, "-r", VIR, "--qi", "--ri"], min_rows=3)


@pytest.mark.parametrize("flags", [[], ["-n", "2"], ["--ci"], ["--detailed"]])
def test_dist_reads_in_blocks(flags):
    _, flushes = same_with_gpus(["dist", "-q", O157, "--qi", "-r"] + FILES + flags, write_count=37, min_rows=200)
    assert len(flushes) >= 5                                                  # blocks of 37 reads


@pytest.fixture(scope="module")
def dbs(tmp_path_factory):
    d = tmp_path_factory.mktemp("dbs")
    db, sep = str(d / "db"), str(d / "sep")
    run(["sketch"] + FILES + ["-o", db])
    run(["sketch"] + FILES + ["-o", sep, "--separate-sketches"])
    return db, sep, [os.path.join(sep, os.path.basename(f) + ".sketch") for f in FILES]


def test_dist_sketch_files(dbs):
    _, sep, sk_files = dbs
    same_with_gpus(["dist", "-q", O157, "--qi", "-r"] + sk_files + [os.path.join(sep, "markers.bin")], write_count=37, min_rows=200)
    same_with_gpus(["dist", "-q"] + sk_files + ["-r"] + sk_files, min_rows=3)
    same_with_gpus(["dist", "-q"] + sk_files + ["-r"] + FILES, min_rows=3)


@pytest.mark.parametrize("layout", ["consolidated", "separate"])
def test_search(dbs, layout):
    db = dbs[0] if layout == "consolidated" else dbs[1]
    # one query per block: a query hits at most two references, so at least one of the three contexts gets no hits
    _, flushes = same_with_gpus(["search", "-d", db] + FILES, write_count=1, min_rows=3)
    assert len(flushes) == 2
    same_with_gpus(["search", "-d", db, VIR, "--qi"], write_count=1, min_rows=0)
    same_with_gpus(["search", "-d", db, O157, "--qi", "-n", "1"], write_count=100, min_rows=0)
    same_with_gpus(["search", "-d", db] + dbs[2], min_rows=3)                 # .sketch queries
    # one reference per import group: every context imports and chains its hits over several rounds
    one = run(["search", "-d", db] + FILES)
    for gpus in ("1", "2"):
        assert run(["search", "-d", db] + FILES + ["--gpus", gpus], env={"SK_SKETCH_GROUP_RECORDS": "1"}) == one
