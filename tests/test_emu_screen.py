"""Host emulation of the marker screen's predicate (skani_b200/csrc/sk_core.cuh: screen_pass, screen_row_rescued) against the
oracle's check_markers_quickly, screen_refs and screen_refs_indices: marker counts 0-25, 105-112, 214-220, 323-330, 1000 and
5000 on either side, shared counts 0, 1, thr - 1, thr, thr + 1 and the full overlap, screen_val 0 (-> 0.80), 0.5, 0.8, 0.95,
0.99 and 1.0, rescue on and off, both argument orders.  See tests/emu/emu_screen.cpp."""
import os
import re
import subprocess

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_screen_predicate_matches_oracle(tmp_path):
    exe = str(tmp_path / "emu_screen")
    subprocess.check_call(["/usr/bin/g++", "-O2", "-std=c++17", "-fopenmp", "-o", exe, os.path.join(ROOT, "tests", "emu", "emu_screen.cpp"),
                           os.path.join(ROOT, "oracle", "skani_oracle.cpp"), "-lz"])
    out = subprocess.run([exe], capture_output=True, text=True, timeout=600)
    assert out.returncode == 0, out.stdout + out.stderr
    m = re.search(r"(\d+) cases, (\d+) on a threshold \((\d+) pass the quick screen and fail screen_refs\), (\d+) rescued rows without a "
                  r"shared marker, (\d+) small columns that do not rescue their row, 0 failures", out.stdout)
    assert m, out.stdout
    cases, on_thr, quick_only, rescued, small_col = map(int, m.groups())
    assert cases > 1_000_000 and on_thr > 0 and quick_only > 0 and rescued > 0 and small_col > 0, out.stdout
