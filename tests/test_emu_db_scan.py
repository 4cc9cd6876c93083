"""CPU: the framing walk of a skani v0.3 sketch entry (skani_b200/cli/sketch_db.hpp: scan_entry, expand_records and
get_sketch built on them) on blobs written by the host writer -- multi-position lists of 2 to 1000 positions, zero keys,
marker-only sketches, zero contigs: the expansion returns the writer's records in order and as many as the scan counts,
every truncation throws without reading past the blob (AddressSanitizer), corrupt length prefixes and Option tags are
refused with the reader's messages, and an out-of-range multi-position index is left to the expansion.  The scan and
expansion are also checked against the independent Python decoder (tests/skani_db_py.py).  See tests/emu/emu_db_scan.cpp."""
import glob
import os
import subprocess
from collections import Counter

import skani_db_py as D

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_scan_entry(tmp_path):
    exe = str(tmp_path / "emu_db_scan")
    subprocess.check_call(["/usr/bin/g++", "-O1", "-g", "-std=c++17", "-fsanitize=address", "-fno-omit-frame-pointer", "-o", exe,
                           os.path.join(ROOT, "tests", "emu", "emu_db_scan.cpp")])
    out_dir = tmp_path / "cases"
    out_dir.mkdir()
    p = subprocess.run([exe, str(out_dir)], capture_output=True, text=True, timeout=600,
                       env=dict(os.environ, ASAN_OPTIONS="detect_leaks=0"))
    assert p.returncode == 0 and "9 cases, 0 failures" in p.stdout, p.stdout + p.stderr
    blobs = sorted(glob.glob(str(out_dir / "case*.sketch")))
    assert len(blobs) == 8
    for path in blobs:
        c = D.Cur(open(path, "rb").read())
        par = D.params(c)
        s = D.sketch(c)
        assert c.o == len(c.b) and (par["c"], par["k"], par["marker_c"]) == (30, 15, 200)
        head, rec = open(path[:-len(".sketch")] + ".txt").read().split("\n")[:2]
        n_keys, n_records, n_multi, n_ctg, n_markers = map(int, head.split()[1:])
        r = list(map(int, rec.split()[1:]))
        got = sorted(zip(r[0::3], r[1::3], r[2::3]), key=lambda x: (x[0], x[2] >> 1, x[1]))
        assert got == s["records"] and n_records == len(s["records"]) and n_keys == s["n_keys"], path
        assert n_ctg == len(s["contig_lengths"]) and n_markers == len(s["markers"])
        per_key = Counter(k for k, _, _ in got)
        assert n_multi == sum(1 for v in per_key.values() if v > 1) and n_keys == len(per_key)
