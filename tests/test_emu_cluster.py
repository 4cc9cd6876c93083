"""sk_cluster's per-vertex logic (skani_b200/csrc/cluster_core.cuh) on the CPU: 2,250 random graphs (Erdos-Renyi, cliques
joined by bridges, paths in rank order and reversed, stars, equal ANIs, ani == min_ani, NaN / -1 / 0.1 rows, isolated
vertices, no genomes).  Host loops emulate the kernels' rounds in three visit orders each (live states in two random
orders, start-of-round states in a third); greedy and single linkage must equal a sequential reference every time.  See
tests/emu/emu_cluster.cpp."""
import os
import re
import subprocess

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_cluster_rounds_match_sequential(tmp_path):
    exe = str(tmp_path / "emu_cluster")
    subprocess.check_call(["/usr/bin/g++", "-O2", "-std=c++17", "-o", exe, os.path.join(ROOT, "tests", "emu", "emu_cluster.cpp")])
    out = subprocess.run([exe], capture_output=True, text=True, timeout=600)
    assert out.returncode == 0, out.stdout + out.stderr
    m = re.search(r"(\d+) cases, (\d+) edges, (\d+) greedy clusters, (\d+) components, (\d+) greedy rounds \((\d+) on rank-ordered paths\), "
                  r"(\d+) hook passes, 0 failures", out.stdout)
    assert m, out.stdout + out.stderr
    cases, edges, greedy, comps, rounds, path_rounds, passes = map(int, m.groups())
    assert cases >= 2000 and edges > 0 and passes > 0
    assert comps < greedy and path_rounds > 0 and rounds > path_rounds, out.stdout
