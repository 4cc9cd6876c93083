"""The row bands and scan tiles of neighbour joining on several contexts (plan_nj, skani_b200/csrc/nj_plan.hpp) on the CPU:
every square of 1 to 400 row tiles over 1 to 16 contexts, more contexts than row tiles included.  The bands cover the row
tiles in order without overlap, every upper-triangle tile is scanned by exactly one context, a context only scans tiles it
holds rows for, and every context's load is within nt / 2 + N tiles of the mean (half a row of tiles).  See tests/emu/emu_nj_plan.cpp."""
import os
import re
import subprocess

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_nj_plan(tmp_path):
    exe = str(tmp_path / "emu_nj_plan")
    subprocess.check_call(["/usr/bin/g++", "-O2", "-std=c++17", "-o", exe, os.path.join(ROOT, "tests", "emu", "emu_nj_plan.cpp")])
    out = subprocess.run([exe], capture_output=True, text=True, timeout=600)
    assert out.returncode == 0, out.stdout + out.stderr
    m = re.search(r"(\d+) cases, (\d+) tiles, (\d+) transposed, (\d+) empty bands, worst load ([\d.]+) of the bound, 0 failures", out.stdout)
    assert m, out.stdout + out.stderr
    cases, tiles, transposed, empty = map(int, m.groups()[:4])
    assert cases == 400 * 16 and tiles > 0 and transposed > 0 and empty > 0, out.stdout
