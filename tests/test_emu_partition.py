"""Pair components and the multi-context pair split of sk_triangle_multi (pair_components, partition_pairs,
skani_b200/csrc/ws_plan.hpp) on the CPU: 3,000 random pair graphs (clustered, one giant component, isolated pairs, no pairs)
over 1 to 12 contexts.  The groups are the components in order of their smallest genome with sorted pairs; every pair lands in
exactly one sorted list, a component of at most cap pairs stays on one context, the split is identical across runs and the
loads differ by at most cap.  See tests/emu/emu_partition.cpp."""
import os
import re
import subprocess

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_pair_partition(tmp_path):
    exe = str(tmp_path / "emu_partition")
    subprocess.check_call(["/usr/bin/g++", "-O2", "-std=c++17", "-o", exe, os.path.join(ROOT, "tests", "emu", "emu_partition.cpp")])
    out = subprocess.run([exe], capture_output=True, text=True, timeout=600)
    assert out.returncode == 0, out.stdout + out.stderr
    m = re.search(r"(\d+) cases, (\d+) pairs, (\d+) components \((\d+) kept whole, (\d+) cut\), (\d+) with more contexts than pairs, "
                  r"0 failures", out.stdout)
    assert m, out.stdout + out.stderr
    cases, pairs, comps, whole, cut, more = map(int, m.groups())
    assert cases == 3000 and pairs > 0 and comps > 0
    assert whole > 0 and cut > 0 and more > 0, out.stdout
