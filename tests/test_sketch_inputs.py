"""CPU: the sketch inputs of `triangle` / `dist` (.sketch files and consolidated databases, skani_b200/cli/sketch_db.hpp:
open_sketch_inputs + SketchGroupReader) through `skani-db-tool groups`, against the independent Python decoder
(tests/skani_db_py.py): genome order (entries in index.db order, merged with loose .sketch files, stably sorted by file
name), per-sketch record counts, the grouping by record count, and the refusals (index entries past the end of
sketches.db, index.db / markers.bin count mismatch, differing parameters, amino-acid databases, undecodable entries)."""
import os
import shutil
import struct
import subprocess

import numpy as np

import oracle_py as O
import skani_db_py as D
from conftest import db_tool


def text_of(name, order, sk):
    e = sk.export()
    lines = ["S %d %d %s" % (order, sk.total_len, name), "C " + name + " contig"]
    lines.append("L %d " % len(e["contig_lengths"]) + " ".join(map(str, e["contig_lengths"].tolist())))
    rec = np.stack([e["kmer"], e["pos"], e["cc"]], 1).reshape(-1)
    lines.append("R %d " % len(e["kmer"]) + " ".join(map(str, rec.tolist())))
    lines.append("M %d " % len(e["markers"]) + " ".join(map(str, e["markers"].tolist())))
    lines.append("E")
    return "\n".join(lines) + "\n"


def write_db(d, genomes, c=30):
    """genomes: [(file name, contig_order, seed)] -> a database written by the CLI's writer"""
    os.makedirs(d)
    text = ""
    for name, order, seed in genomes:
        g = np.random.default_rng(seed).choice(np.frombuffer(b"ACGT", np.uint8), 20_000 + 3_000 * (seed % 7))
        text += text_of(name, order, O.sketch_from_contigs(name, [g], c=c, k=15, marker_c=200))
    subprocess.run([db_tool(), "write", d, str(c), "15", "200"], input=text.encode(), check=True)
    return d


def groups(args, bound=10 ** 9, threads=2):
    p = subprocess.run([db_tool(), "groups", str(bound), str(threads)] + args, capture_output=True, text=True)
    return p.returncode, p.stdout, p.stderr


def parse(out):
    lines = out.splitlines()
    assert lines[0].startswith("PARAMS ") and lines[1].startswith("N ")
    gs, sk = [], []
    for ln in lines[2:]:
        t = ln.split(" ", 3)
        if t[0] == "G":
            gs.append((int(t[1]), int(t[2]), int(t[3])))
        else:
            sk.append((t[3], int(t[1]), int(t[2])))
    assert len(sk) == int(lines[1].split()[1]) and sum(g[1] for g in gs) == len(sk)
    return [int(x) for x in lines[0].split()[1:]], gs, sk


def expected_groups(recs, bound):
    """greedy cut: a group takes sketches while its records stay < bound; every group holds at least one sketch"""
    out, first, acc = [], 0, 0
    for i, r in enumerate(recs):
        if i > first and acc + r >= bound:
            out.append((first, i - first, acc))
            first, acc = i, 0
        acc += r
    if recs:
        out.append((first, len(recs) - first, acc))
    return out


def setup(tmp_path):
    a = write_db(str(tmp_path / "a"), [("g/b.fa", 0, 1), ("g/d.fa", 0, 2), ("g/a.fa", 0, 3), ("g/same.fa", 0, 4)])
    b = write_db(str(tmp_path / "b"), [("g/same.fa", 1, 5), ("g/c.fa", 0, 6), ("g/e.fa", 0, 7)])
    # a loose .sketch file: one (SketchParams, Sketch) blob, here cut out of a third database
    c = write_db(str(tmp_path / "c"), [("g/bb.fa", 0, 8)])
    name, off, ln = D.read_db(c)[3][0]
    sk = str(tmp_path / "bb.fa.sketch")
    open(sk, "wb").write(open(os.path.join(c, "sketches.db"), "rb").read()[off:off + ln])
    return a, b, sk


def decoded(d):
    return [(s["file_name"], len(s["records"]), s["contig_order"]) for s in D.read_db(d)[1]]


def test_order_records_and_groups(tmp_path):
    a, b, sk = setup(tmp_path)
    # entries in index.db order per input, inputs in command-line order, then a stable sort by file name
    merged = decoded(a) + [decoded(str(tmp_path / "c"))[0]] + decoded(b)
    want = sorted(merged, key=lambda x: x[0])
    assert [w[0] for w in want].count("g/same.fa") == 2
    rc, out, err = groups([a, sk, b])
    assert rc == 0, err
    par, gs, got = parse(out)
    assert par == [30, 15, 200]
    assert got == want and gs == [(0, len(want), sum(w[1] for w in want))]
    assert [g[2] for g in got if g[0] == "g/same.fa"] == [0, 1]          # a's entry first: a comes first on the command line
    # markers.bin next to loose .sketch files is skipped, as in file_io::sketches_from_sketch
    shutil.copy(os.path.join(a, "markers.bin"), str(tmp_path / "markers.bin"))
    assert parse(groups([b, str(tmp_path / "markers.bin"), sk, a])[1])[2] == sorted(decoded(b) + merged[4:5] + decoded(a), key=lambda x: x[0])
    # many groups: every bound from one sketch per group to all in one, with 1 and 4 threads
    recs = [w[1] for w in want]
    for bound in (1, min(recs), 2 * min(recs) + 1, sum(recs) // 3, sum(recs), sum(recs) + 1):
        for threads in (1, 4):
            rc, out, err = groups([a, sk, b], bound, threads)
            assert rc == 0, err
            _, gs, got = parse(out)
            assert got == want and gs == expected_groups(recs, bound), (bound, threads)
    assert len(expected_groups(recs, 2 * min(recs) + 1)) > 3


def test_refusals(tmp_path):
    a, b, sk = setup(tmp_path)

    def refused(args, text):
        rc, out, err = groups(args)
        assert rc == 1 and text in err, err

    # an index entry running past the end of a truncated sketches.db
    t = str(tmp_path / "trunc")
    shutil.copytree(a, t)
    raw = open(os.path.join(t, "sketches.db"), "rb").read()
    open(os.path.join(t, "sketches.db"), "wb").write(raw[:len(raw) - 100])
    refused([b, t], "ERROR Failed to load consolidated database: the entry of g/same.fa runs past the end of")
    # index.db and markers.bin disagree on the number of sketches
    m = str(tmp_path / "mism")
    shutil.copytree(a, m)
    mb = bytearray(open(os.path.join(m, "markers.bin"), "rb").read())
    n = struct.unpack_from("<Q", mb, 626)[0]
    struct.pack_into("<Q", mb, 626, n + 1)
    open(os.path.join(m, "markers.bin"), "wb").write(bytes(mb))
    refused([m], "ERROR index.db and markers.bin disagree on the number of sketches")
    # without markers.bin the index alone describes the database
    os.remove(os.path.join(m, "markers.bin"))
    assert parse(groups([m])[1])[2] == sorted(decoded(a), key=lambda x: x[0])
    # different parameters: both inputs named
    c125 = write_db(str(tmp_path / "c125"), [("g/x.fa", 0, 9)], c=125)
    refused([a, c125], "ERROR Sketch parameters of %s (c = 125, k = 15, m = 200) differ from those of %s (c = 30, k = 15, m = 200)" % (c125, a))
    refused([sk, c125], "differ from those of %s" % sk)
    # an amino-acid database: the use_aa byte of SketchParams (after c, k, marker_c and use_syncs) in the first entry
    aa = str(tmp_path / "aa")
    shutil.copytree(a, aa)
    for f in ("sketches.db", "markers.bin"):
        raw = bytearray(open(os.path.join(aa, f), "rb").read())
        raw[25] = 1
        open(os.path.join(aa, f), "wb").write(bytes(raw))
    refused([aa], "ERROR amino-acid databases are not supported")
    # an entry that does not decode (the second one: the first is decoded when the database is opened)
    bad = str(tmp_path / "bad")
    shutil.copytree(a, bad)
    name, off, ln = D.read_db(a)[3][1]
    raw = bytearray(open(os.path.join(bad, "sketches.db"), "rb").read())
    raw[off + 626:off + 634] = (2 ** 60).to_bytes(8, "little")          # the file-name length prefix
    open(os.path.join(bad, "sketches.db"), "wb").write(bytes(raw))
    rc, out, err = groups([bad])
    assert rc == 1 and "ERROR Failed to load sketch %s" % name in err
