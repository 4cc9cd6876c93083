"""Host emulation of the chain front end's compacted hit stream (probe_kernel's per-tile hit lists and counted bits, the
tiles' hit offsets, chunk_anchor_kernel stepping over 1,024 hits at a time with carries) against the oracle's chunk
boundaries on 40 ordered pairs (c in {125, 30}) and against a plain record-order pass on constructed hit patterns: a step
whose hits span many tiles with runs of hit-free tiles, a tile in which every record hits, a pair whose only hit is its
last record, hit counts on and off a multiple of 1,024, a contig boundary on a step boundary, a record with `band` anchors
at the end of a step.  See tests/emu/emu_chain_hits.cpp."""
import os
import re
import subprocess

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_chain_hit_stream_matches_oracle(tmp_path):
    exe = str(tmp_path / "emu_chain_hits")
    subprocess.check_call(["/usr/bin/g++", "-O2", "-std=c++17", "-fopenmp", "-o", exe,
                           os.path.join(ROOT, "tests", "emu", "emu_chain_hits.cpp"), os.path.join(ROOT, "oracle", "skani_oracle.cpp"), "-lz"])
    out = subprocess.run([exe], capture_output=True, text=True, timeout=600)
    assert out.returncode == 0, out.stdout + out.stderr
    m = re.search(r"(\d+) oracle pairs, (\d+) constructed pairs, 0 failures", out.stdout)
    assert m and int(m.group(1)) == 40 and int(m.group(2)) == 6, out.stdout
    t = re.search(r"steps (\d+) \((\d+) over several tiles, (\d+) hit-free tiles passed\), full tiles (\d+), contig on step "
                  r"boundary (\d+), straddling: step (\d+) round (\d+), H multiple of TILE (\d+) / not (\d+)", out.stdout)
    assert t and all(int(x) > 0 for x in t.groups()), out.stdout
