"""GPU: `skani-b200 sketch` writes its database from entries encoded on the device.  The directories it writes
(sketches.db, index.db, markers.bin, and the .sketch files with --separate-sketches) are byte-identical to the host
writer's (skani-db-tool write) for the same sketches, and identical across --gpus 1 and --gpus 3 (contexts sharing one
device), one group and many forced groups (SK_SKETCH_GROUP_FILES), with and without -i, and at -c 30.  The inputs hold
more than 100 genomes, so the progress lines are written.  `triangle DB` on a database written with --gpus 2 prints what
`triangle` prints on the FASTA files, and an existing output directory is still refused."""
import os
import subprocess

import numpy as np
import pytest

from conftest import db_tool

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
BIN = os.path.join(ROOT, "skani_b200", "skani-b200")
GOLD = os.path.join(ROOT, "tests", "golden")


def cli(args, env=None):
    e = {k: v for k, v in os.environ.items() if not k.startswith("SK_")}
    e.update(env or {})
    p = subprocess.run([BIN] + args, capture_output=True, text=True, timeout=900, env=e)
    assert p.returncode == 0, p.stderr
    return p


@pytest.fixture(scope="module")
def inputs(tmp_path_factory):
    """120 synthetic genomes in 40 families (so that triangle has pairs to report), plus the golden E. coli and viruses"""
    d = tmp_path_factory.mktemp("fa")
    rng = np.random.default_rng(3)
    acgt = np.frombuffer(b"ACGT", np.uint8)
    files = []
    for f in range(40):
        base = acgt[rng.integers(0, 4, 60000)]
        for m in range(3):
            g = base.copy()
            flip = rng.random(len(g)) < 0.01 * m
            g[flip] = acgt[rng.integers(0, 4, int(flip.sum()))]
            p = str(d / ("fam%02d_m%d.fa" % (f, m)))
            with open(p, "wb") as fh:
                fh.write(b">%s contig one\n" % os.path.basename(p).encode() + g[:35000].tobytes() + b"\n>second\n" + g[35000:].tobytes() + b"\n")
            files.append(p)
    return files + [os.path.join(GOLD, f) for f in ("e.coli-EC590.fasta.gz", "e.coli-K12.fasta.gz", "viruses.fna")]


def tree(d):
    return {f: open(os.path.join(d, f), "rb").read() for f in sorted(os.listdir(d))}


def host_rewrite(db, out, c, m):
    """the host writer's database for the sketches of db (read back by skani-db-tool dump)"""
    text = subprocess.run([db_tool(), "dump", db], capture_output=True, text=True, check=True).stdout
    text = text.split("\nK ", 1)[0] + "\n"
    os.makedirs(out)
    subprocess.run([db_tool(), "write", out, str(c), "15", str(m)], input=text, text=True, check=True)
    return tree(out)


@pytest.mark.parametrize("flags,c,m", [([], 125, 1000), (["-i"], 125, 1000), (["-c", "30"], 30, 1000)], ids=["plain", "individual", "c30"])
def test_sketch_db_bytes(tmp_path, inputs, flags, c, m):
    runs = {}
    for name, gpus, env in (("one", 1, None), ("three", 3, None), ("groups", 1, {"SK_SKETCH_GROUP_FILES": "7"}),
                            ("groups3", 3, {"SK_SKETCH_GROUP_FILES": "7"})):
        out = str(tmp_path / name)
        p = cli(["sketch"] + inputs + flags + ["-o", out, "--gpus", str(gpus), "-t", "4"], env)
        assert "sequences sketched." in p.stderr and "INFO Successfully wrote" in p.stderr
        assert "sketches written in %d group(s)" % (1 if env is None else -(-len(inputs) // 7)) in p.stderr
        runs[name] = tree(out)
    assert set(runs["one"]) == {"sketches.db", "index.db", "markers.bin"}
    for name in ("three", "groups", "groups3"):
        assert runs[name] == runs["one"], name
    assert host_rewrite(str(tmp_path / "one"), str(tmp_path / "host"), c, m) == runs["one"]


@pytest.mark.parametrize("flags", [[], ["-i"]], ids=["plain", "individual"])
def test_separate_sketches(tmp_path, inputs, flags):
    db = str(tmp_path / "db")
    cli(["sketch"] + inputs + flags + ["-o", db])
    want = tree(db)
    sep = {}
    for gpus, env in ((1, None), (3, {"SK_SKETCH_GROUP_FILES": "5"})):
        out = str(tmp_path / ("sep%d" % gpus))
        cli(["sketch"] + inputs + flags + ["-o", out, "--separate-sketches", "--gpus", str(gpus)], env)
        sep[gpus] = tree(out)
    assert sep[1] == sep[3]
    assert sep[1]["markers.bin"] == want["markers.bin"]
    # each .sketch file is the database's entry of the same sketch
    entries = sorted(v for k, v in sep[1].items() if k.endswith(".sketch"))
    idx = open(os.path.join(db, "index.db"), "rb").read()
    n = int.from_bytes(idx[:8], "little")
    o, blobs = 8, []
    for _ in range(n):
        ln = int.from_bytes(idx[o:o + 8], "little"); o += 8 + ln
        off, size = int.from_bytes(idx[o:o + 8], "little"), int.from_bytes(idx[o + 8:o + 16], "little"); o += 16
        blobs.append(want["sketches.db"][off:off + size])
    assert len(entries) == n and entries == sorted(blobs)
    if flags:
        assert any(k.startswith("1_") for k in sep[1])


def test_triangle_on_multi_gpu_db(tmp_path, inputs):
    db = str(tmp_path / "db")
    cli(["sketch"] + inputs + ["-o", db, "--gpus", "2"])
    want = cli(["triangle"] + inputs + ["-E"]).stdout
    got = cli(["triangle", db, "-E"]).stdout
    assert got == want and len(want.splitlines()) > 40
    p = subprocess.run([BIN, "sketch", inputs[0], "-o", db], capture_output=True, text=True)
    assert p.returncode != 0 and "Output directory exists" in p.stderr
