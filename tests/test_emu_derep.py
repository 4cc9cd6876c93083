"""Host emulation of sk_dereplicate's oriented screen predicate (skani_b200/csrc/derep_core.cuh: dr_screen_pass) against the
oracle's screen_refs as the triangle applies it (the smaller genome index is the query): wave genome below and above the
representative, either argument order, marker counts 0, 19, 20, 21, 30, 107 and 1000 on either side, shared counts 0, 1,
thr - 1, thr, thr + 1 and the full overlap, rescue on and off.  See tests/emu/emu_derep.cpp."""
import os
import re
import subprocess

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_oriented_predicate_matches_oracle(tmp_path):
    exe = str(tmp_path / "emu_derep")
    subprocess.check_call(["/usr/bin/g++", "-O2", "-std=c++17", "-fopenmp", "-o", exe, os.path.join(ROOT, "tests", "emu", "emu_derep.cpp"),
                           os.path.join(ROOT, "oracle", "skani_oracle.cpp"), "-lz"])
    out = subprocess.run([exe], capture_output=True, text=True, timeout=600)
    assert out.returncode == 0, out.stdout + out.stderr
    m = re.search(r"(\d+) cases, (\d+) on a threshold, (\d+) rescued by the smaller index, (\d+) small larger indices not rescued, "
                  r"0 failures", out.stdout)
    assert m, out.stdout
    cases, on_thr, rescued, not_rescued = map(int, m.groups())
    assert cases > 1000 and on_thr > 0 and rescued > 0 and not_rescued > 0, out.stdout
