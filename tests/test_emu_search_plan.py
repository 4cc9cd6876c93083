"""search's query-group plan (skani_b200/cli/search_plan.hpp) on the CPU: the streaming name ranks, which need only the
reference names, order every (reference, query) pair as dense ranks over all names together do (random name sets with equal
names, names between references, before the first and after the last), and the group cutter covers every query once and in
order, keeps groups within the file and bases bounds, and splits a file only with --qi when it alone exceeds the bases bound.
See tests/emu/emu_search_plan.cpp."""
import os
import re
import subprocess

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_search_plan(tmp_path):
    exe = str(tmp_path / "emu_search_plan")
    subprocess.check_call(["/usr/bin/g++", "-O2", "-std=c++17", "-o", exe, os.path.join(ROOT, "tests", "emu", "emu_search_plan.cpp")])
    out = subprocess.run([exe], capture_output=True, text=True, timeout=600)
    assert out.returncode == 0, out.stdout + out.stderr
    m = re.search(r"(\d+) rank pairs \((\d+) equal, (\d+) before, (\d+) after\), (\d+) cut cases, (\d+) groups, (\d+) split files, 0 failures",
                  out.stdout)
    assert m, out.stdout
    pairs, equal, before, after, cases, groups, split = map(int, m.groups())
    assert pairs > 10000 and equal > 100 and before > 1000 and after > 1000
    assert cases == 3000 and groups > cases and split > 50
