"""`skani-b200 triangle` / `dist` with consolidated sketch databases (folders written by `sketch`: sketches.db, index.db,
markers.bin) as inputs, alone or mixed with .sketch files: stdout (and the .af matrix where one is written) must equal
the run on the FASTA inputs, and on their --separate-sketches .sketch files, byte for byte -- on the in-memory path, on
the store path (a small SK_DEVICE_BUDGET_MB), with the input cut into many groups (SK_SKETCH_GROUP_RECORDS) and with
--gpus 3 on one device.  Refused inputs end with an ERROR line and exit 1."""
import os
import shutil
import struct
import subprocess

import pytest

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
BIN = os.path.join(ROOT, "skani_b200", "skani-b200")
GOLD = os.path.join(ROOT, "tests", "golden")
EC, K12, VIR, TEST, O157 = (os.path.join(GOLD, f) for f in ("e.coli-EC590.fasta.gz", "e.coli-K12.fasta.gz", "viruses.fna", "test.fasta",
                                                            "o157_reads.fa.gz"))
FILES = [EC, K12, VIR, TEST]
STORE = {"SK_DEVICE_BUDGET_MB": "8"}                              # about 2 MB per E. coli sketch: several working sets
GROUPS = {"SK_DEVICE_BUDGET_MB": "8", "SK_SKETCH_GROUP_RECORDS": "3000"}   # and about one sketch per import group
MEM_GROUPS = {"SK_SKETCH_GROUP_RECORDS": "3000"}                 # in memory: one set grown by sk_sketch_set_append


def cli(args, cwd, env=None, rc=0):
    e = {k: v for k, v in os.environ.items() if k not in ("SK_DEVICE_BUDGET_MB", "SK_SKETCH_GROUP_RECORDS")}
    e.update(env or {})
    os.makedirs(cwd, exist_ok=True)
    af = os.path.join(cwd, "skani_matrix.af")
    if os.path.exists(af):
        os.remove(af)
    p = subprocess.run([BIN] + args, capture_output=True, text=True, timeout=900, env=e, cwd=cwd)
    assert p.returncode == rc, p.stderr
    return p.stdout, open(af).read() if os.path.exists(af) else None, p.stderr


@pytest.fixture(scope="module")
def dbs(tmp_path_factory):
    d = tmp_path_factory.mktemp("dbs")
    out = {}

    def sketch(name, args):
        out[name] = str(d / name)
        cli(["sketch"] + args + ["-o", out[name]], str(d))

    sketch("all", FILES)
    sketch("sep", FILES + ["--separate-sketches"])
    sketch("ind", [VIR, TEST, EC, "-i"])
    sketch("reads", [O157, "-i"])
    sketch("part1", [EC, TEST])
    sketch("part2", [K12])
    sketch("c30", [VIR, "-c", "30"])
    out["sketches"] = [os.path.join(out["sep"], os.path.basename(f) + ".sketch") for f in (EC, K12, VIR)]   # test.fasta: < 500 bp
    return out


MODES = {"matrix": [], "sparse": ["-E"], "full_matrix": ["--full-matrix"], "distance": ["--distance", "--full-matrix"],
         "diagonal": ["--diagonal"], "sparse_detailed": ["-E", "--detailed", "--diagonal"]}


def same(runs, min_lines=2):
    first = runs[0]
    for r in runs[1:]:
        assert r[0] == first[0] and r[1] == first[1]
    assert len(first[0].strip().split("\n")) >= min_lines
    return first


@pytest.mark.parametrize("mode", sorted(MODES))
def test_triangle_db_equals_fasta_and_sketch_files(dbs, tmp_path, mode):
    f = MODES[mode]
    fasta = cli(["triangle"] + FILES + f, str(tmp_path))
    db = cli(["triangle", dbs["all"]] + f, str(tmp_path))
    assert "INFO Sketches detected" in db[2] and "INFO 3 sketches loaded in 1 group(s)" in db[2]
    same([fasta, db, cli(["triangle"] + dbs["sketches"] + f, str(tmp_path))])
    assert (fasta[1] is None) == ("-E" in f)
    # the store path, and the store path with about one sketch per import group
    st = cli(["triangle", dbs["all"]] + f, str(tmp_path), STORE)
    gr = cli(["triangle", dbs["all"]] + f, str(tmp_path), GROUPS)
    assert "INFO Store path" in st[2] and "INFO 3 sketches loaded in 3 group(s)" in gr[2]
    same([fasta, st, gr])


def test_triangle_individual(dbs, tmp_path):
    for f in ([], ["-E"]):
        fasta = cli(["triangle", VIR, TEST, EC, "-i"] + f, str(tmp_path))
        runs = [cli(["triangle", dbs["ind"], "-i"] + f, str(tmp_path), env) for env in (None, STORE, GROUPS)]
        same([fasta] + runs)


def test_triangle_several_inputs(dbs, tmp_path):
    """two databases plus a loose .sketch file: the genome order and output of one database holding all of them"""
    loose = dbs["sketches"][2]
    for f in ([], ["-E", "--ci"]):
        one = cli(["triangle", dbs["all"]] + f, str(tmp_path))
        for env in (None, GROUPS):
            same([one, cli(["triangle", dbs["part2"], loose, dbs["part1"]] + f, str(tmp_path), env)])
    # the list file (-l) takes databases too
    lst = tmp_path / "list.txt"
    lst.write_text("\n".join([dbs["part1"], dbs["part2"], loose]) + "\n")
    same([cli(["triangle", "-E", dbs["all"]], str(tmp_path)), cli(["triangle", "-E", "-l", str(lst)], str(tmp_path))])


DIST = {"plain": [], "n2": ["-n", "2"], "ci": ["--ci"], "detailed": ["--detailed"]}


@pytest.mark.parametrize("flags", sorted(DIST))
def test_dist(dbs, tmp_path, flags):
    f = DIST[flags]
    t = str(tmp_path)
    # -q FASTA -r DB, and one database on both sides
    want = cli(["dist", "-q", EC, K12, "-r"] + FILES + f, t)
    for env in (None, STORE, GROUPS):
        same([want, cli(["dist", "-q", EC, K12, "-r", dbs["all"]] + f, t, env)], min_lines=3)
    want = cli(["dist", "-q"] + FILES + ["-r"] + FILES + f, t)
    for env in (None, STORE, GROUPS):
        same([want, cli(["dist", "-q", dbs["all"], "-r", dbs["all"]] + f, t, env),
              cli(["dist", "-q"] + dbs["sketches"] + ["-r", dbs["part1"], dbs["part2"], dbs["sketches"][2]] + f, t, env)], min_lines=5)
    # --qi queries from a database sketched with -i (the reads), against FASTA and against database references
    want = cli(["dist", "-q", O157, "--qi", "-r", EC, K12] + f, t)
    for env in (None, STORE):
        same([want, cli(["dist", "-q", dbs["reads"], "--qi", "-r", EC, K12] + f, t, env),
              cli(["dist", "-q", dbs["reads"], "--qi", "-r", dbs["part1"], dbs["part2"]] + f, t, env)], min_lines=100)


def test_dist_lists(dbs, tmp_path):
    """--ql / --rl list files name databases as well"""
    ql, rl = tmp_path / "ql.txt", tmp_path / "rl.txt"
    ql.write_text(dbs["reads"] + "\n")
    rl.write_text(dbs["part1"] + "\n" + dbs["part2"] + "\n")
    t = str(tmp_path / "run")
    same([cli(["dist", "-q", O157, "--qi", "-r", EC, K12], t), cli(["dist", "--ql", str(ql), "--qi", "--rl", str(rl)], t)], min_lines=100)


def test_gpus_3_on_one_device(dbs, tmp_path):
    t = str(tmp_path)
    for args in (["triangle", dbs["all"]], ["triangle", "-E", dbs["all"]], ["triangle"] + dbs["sketches"], ["triangle", dbs["ind"], "-i"]):
        one = cli(args, t)
        three = cli(args + ["--gpus", "3"], t)
        assert "INFO Store path" in three[2] and "on 3 GPU(s)" in three[2] and "INFO Store path" not in one[2]
        same([one, three])
    for args in (["dist", "-q", EC, K12, "-r", dbs["all"]], ["dist", "-q", dbs["reads"], "--qi", "-r", dbs["all"]]):
        one = cli(args, t)
        same([one, cli(args + ["--gpus", "3"], t), cli(args + ["--gpus", "3"], t, STORE)])


def test_refused(dbs, tmp_path):
    t = str(tmp_path / "run")

    def refused(args, text):
        _, _, err = cli(args, t, rc=1)
        assert text in err, err
        assert "INFO Store path" not in err

    refused(["triangle", dbs["all"], EC], "ERROR Sketch database %s cannot be mixed with FASTA/FASTQ inputs" % dbs["all"])
    refused(["dist", "-q", EC, "-r", K12, dbs["all"]], "cannot be mixed with FASTA/FASTQ inputs")
    refused(["triangle", dbs["all"], dbs["c30"]], "ERROR Sketch parameters of %s (c = 30, k = 15, m = 1000) differ from those of %s (c = 125" % (dbs["c30"], dbs["all"]))
    refused(["dist", "-q", EC, "-r", dbs["sketches"][0], dbs["c30"]], "differ from those of %s" % dbs["sketches"][0])
    # a truncated sketches.db: the last index entry runs past its end
    trunc = str(tmp_path / "trunc")
    shutil.copytree(dbs["all"], trunc)
    raw = open(os.path.join(trunc, "sketches.db"), "rb").read()
    open(os.path.join(trunc, "sketches.db"), "wb").write(raw[:-1000])
    refused(["triangle", trunc], "ERROR Failed to load consolidated database: the entry of %s runs past the end" % sorted(FILES)[-1])
    refused(["dist", "-q", EC, "-r", trunc], "runs past the end")
    # index.db and markers.bin disagree on the number of sketches
    mism = str(tmp_path / "mism")
    shutil.copytree(dbs["all"], mism)                    # 3 sketches, markers.bin of 1
    shutil.copy(os.path.join(dbs["part2"], "markers.bin"), os.path.join(mism, "markers.bin"))
    refused(["triangle", mism], "ERROR index.db and markers.bin disagree on the number of sketches")
    # an amino-acid database: use_aa, the byte after c, k, marker_c (u64) and use_syncs, set in the first entry and markers.bin
    aa = str(tmp_path / "aa")
    shutil.copytree(dbs["all"], aa)
    for f in ("sketches.db", "markers.bin"):
        raw = bytearray(open(os.path.join(aa, f), "rb").read())
        assert struct.unpack_from("<QQQBB", raw, 0)[3:] == (0, 0)
        raw[25] = 1
        open(os.path.join(aa, f), "wb").write(bytes(raw))
    refused(["triangle", aa], "ERROR amino-acid databases are not supported")
    refused(["dist", "-q", aa, "-r", EC], "ERROR amino-acid databases are not supported")


def test_in_memory_many_groups(dbs, tmp_path):
    """about one sketch per import group on the in-memory path: the groups are appended into one set (one per context with
    dist --gpus 3)"""
    t = str(tmp_path)
    for f in ([], ["-E"]):
        want = cli(["triangle"] + FILES + f, t)
        got = cli(["triangle", dbs["all"]] + f, t, MEM_GROUPS)
        assert "INFO Store path" not in got[2] and "INFO 3 sketches loaded in 3 group(s)" in got[2]
        same([want, got])
    want = cli(["dist", "-q", O157, "--qi", "-r"] + FILES, t)
    for gpus in ([], ["--gpus", "3"]):
        got = cli(["dist", "-q", dbs["reads"], "--qi", "-r", dbs["all"]] + gpus, t, MEM_GROUPS)
        assert "INFO Store path" not in got[2] and "group(s)" in got[2]
        same([want, got], min_lines=100)
    got = cli(["dist", "-q", EC, K12, "-r", dbs["all"], "--gpus", "3"], t, MEM_GROUPS)
    same([cli(["dist", "-q", EC, K12, "-r"] + FILES, t), got])


def test_entry_that_does_not_decode(dbs, tmp_path):
    """only a database's first entry is decoded when it is opened: a later entry that does not decode ends the run while
    the sketches are loaded -- after earlier groups were imported, on every path -- with its ERROR line and exit 1"""
    bad = str(tmp_path / "bad")
    shutil.copytree(dbs["all"], bad)
    ix = open(os.path.join(bad, "index.db"), "rb").read()
    names, o = [], 8
    for _ in range(struct.unpack_from("<Q", ix, 0)[0]):
        n = struct.unpack_from("<Q", ix, o)[0]
        names.append((ix[o + 8:o + 8 + n].decode(), struct.unpack_from("<Q", ix, o + 8 + n)[0]))
        o += 8 + n + 16
    name, off = names[1]                                   # K12: the second entry
    assert name == K12
    raw = bytearray(open(os.path.join(bad, "sketches.db"), "rb").read())
    raw[off + 626:off + 634] = (2 ** 60).to_bytes(8, "little")      # its file-name length prefix
    open(os.path.join(bad, "sketches.db"), "wb").write(bytes(raw))
    t = str(tmp_path / "run")
    for args, env in ((["triangle", bad], None), (["triangle", bad], MEM_GROUPS), (["triangle", bad], GROUPS),
                      (["triangle", bad, "--gpus", "3"], None), (["dist", "-q", EC, "-r", bad], MEM_GROUPS),
                      (["dist", "-q", EC, "-r", bad, "--gpus", "3"], None), (["dist", "-q", EC, "-r", bad], STORE),
                      (["dist", "-q", bad, "-r", EC], None)):
        out, _, err = cli(args, t, env, rc=1)
        assert "ERROR Failed to load sketch %s" % K12 in err, (args, env, err)
        assert "Ref_file" not in out and "INFO Screen + chain" not in err
