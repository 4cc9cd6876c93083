"""Query x reference working-set planner of sk_query_ref_store (plan_query_ref_working_sets, skani_b200/csrc/ws_plan.hpp) on
the CPU: 2,500 random bipartite pair graphs (clustered, one query hitting every reference, every query hitting one reference,
skewed genome sizes, few queries against many references) and budgets from "everything fits" down to twice the largest
genome.  Every pair lands in exactly one working set, reference and query lists are ascending, in range and exactly the
pairs' genomes, working sets stay within the budget, the plan is identical across runs, a genome over budget / 2 on either
side is refused, and one query against many references gathers every reference once.  See tests/emu/emu_qr_plan.cpp."""
import os
import re
import subprocess

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_query_ref_working_set_plan(tmp_path):
    exe = str(tmp_path / "emu_qr_plan")
    subprocess.check_call(["/usr/bin/g++", "-O2", "-std=c++17", "-o", exe, os.path.join(ROOT, "tests", "emu", "emu_qr_plan.cpp")])
    out = subprocess.run([exe], capture_output=True, text=True, timeout=600)
    assert out.returncode == 0, out.stdout + out.stderr
    m = re.search(r"(\d+) cases, (\d+) pairs, (\d+) working sets \((\d+) chunk pairs\), (\d+) split components, "
                  r"(\d+) single-gather checks, (\d+) refusals, 0 failures", out.stdout)
    assert m, out.stdout + out.stderr
    cases, pairs, sets, chunk, split, once, refused = map(int, m.groups())
    assert cases == 2500 and pairs > 0 and refused == 2 * cases
    assert chunk > 0 and split > 0 and sets > chunk and once > 20, out.stdout
