"""sk_cluster_linkage's per-cluster logic (skani_b200/csrc/linkage_core.cuh) on the CPU: 2,400 random graphs (Erdos-Renyi,
cliques joined by bridges, paths, stars, ten ANI values, equal ANIs, ani == min_ani with NaN / -1 / 0.1 rows, dense graphs
for complete linkage's full pairs, isolated genomes, n = 0 / 1), both methods, cut and dendrogram mode.  Host loops emulate
the kernels' rounds in four visit orders (forward, reverse, random, the warp's lane-strided fold); they must agree, the cut
and dendrogram modes must partition alike, and on graphs without ties the merges must equal a sequential HAC.  See
tests/emu/emu_linkage.cpp."""
import os
import re
import subprocess

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_linkage_rounds_match_sequential(tmp_path):
    exe = str(tmp_path / "emu_linkage")
    subprocess.check_call(["/usr/bin/g++", "-O2", "-std=c++17", "-o", exe, os.path.join(ROOT, "tests", "emu", "emu_linkage.cpp")])
    out = subprocess.run([exe], capture_output=True, text=True, timeout=600)
    assert out.returncode == 0, out.stdout + out.stderr
    m = re.search(r"(\d+) cases \((\d+) complete linkage\), (\d+) merges, (\d+) rounds, (\d+) checked against sequential HAC, 0 failures", out.stdout)
    assert m, out.stdout + out.stderr
    cases, complete, merges, rounds, hac = map(int, m.groups())
    assert cases >= 2000 and 0 < complete < cases and merges > rounds > 0 and hac >= 1000, out.stdout
