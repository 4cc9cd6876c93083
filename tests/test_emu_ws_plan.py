"""Working-set planner of sk_triangle_store (skani_b200/csrc/ws_plan.hpp) on the CPU: 2,000 random pair graphs (clustered,
one giant component, mostly isolated genomes, skewed genome sizes) and budgets from "everything fits" down to twice the
largest genome.  Every pair lands in exactly one working set, working sets stay within the budget, the plan is identical
across runs, chunk pairs appear exactly for components over budget, and a genome over budget / 2 is refused.  See
tests/emu/emu_ws_plan.cpp."""
import os
import re
import subprocess

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_working_set_plan(tmp_path):
    exe = str(tmp_path / "emu_ws_plan")
    subprocess.check_call(["/usr/bin/g++", "-O2", "-std=c++17", "-o", exe, os.path.join(ROOT, "tests", "emu", "emu_ws_plan.cpp")])
    out = subprocess.run([exe], capture_output=True, text=True, timeout=600)
    assert out.returncode == 0, out.stdout + out.stderr
    m = re.search(r"(\d+) cases, (\d+) pairs, (\d+) working sets \((\d+) chunk pairs, (\d+) packing several components\), "
                  r"(\d+) split components, (\d+) refusals, 0 failures", out.stdout)
    assert m, out.stdout + out.stderr
    cases, pairs, sets, chunk, multi, split, refused = map(int, m.groups())
    assert cases == 2000 and pairs > 0 and refused > 1000
    assert chunk > 0 and split > 0 and multi > 0 and sets > chunk, out.stdout
