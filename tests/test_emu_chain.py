"""Host emulation of the chaining kernels' per-item logic (skani_b200/csrc/chain_core.cuh: chunk-assignment closed form,
interval order + greedy non-overlap filter, random-access WyRand/Lemire, flattened GBDT) against the oracle's parity taps:
7 genome shapes (plain, divergent, anchor-free gaps of 90/65/24 kb, 12 contigs with reverse complements and a repeat, two
repeat-rich genomes, an anchor-free stretch longer than one tile) x c in {125, 30}, all ordered pairs.  The chunk assignment
also runs in chunk_anchor_kernel's own arrangement (1,024-record tiles with carries, the block scans' operator order, random
bracketings).  See tests/emu/emu_chain.cpp."""
import os
import re
import subprocess

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_chain_logic_matches_oracle(tmp_path):
    exe = str(tmp_path / "emu_chain")
    subprocess.check_call(["/usr/bin/g++", "-O2", "-std=c++17", "-fopenmp", "-o", exe, os.path.join(ROOT, "tests", "emu", "emu_chain.cpp"),
                           os.path.join(ROOT, "oracle", "skani_oracle.cpp"), "-lz"])
    out = subprocess.run([exe], capture_output=True, text=True, timeout=600)
    assert out.returncode == 0, out.stdout + out.stderr
    m = re.search(r"(\d+) pairs, (\d+) chunks, (\d+) intervals, (\d+) catch-up anchors, 0 failures", out.stdout)
    assert m and int(m.group(1)) == 84 and int(m.group(2)) > 1000 and int(m.group(3)) > 1000 and int(m.group(4)) > 0, out.stdout
    t = re.search(r"tiles (\d+) \((\d+) without anchors, (\d+) with several rounds\), rounds (\d+), straddling records (\d+), "
                  r"bracketings (\d+), pairs at the chunk bound (\d+)", out.stdout)
    assert t and all(int(x) > 0 for x in t.groups()), out.stdout
