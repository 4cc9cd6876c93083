"""The sketch-set array table (skani_b200/csrc/set_layout.hpp) on the CPU: blob layout, metadata encoder / decoder, sentinel
index rule and the store's genome bytes over random counts, zeros included; see tests/emu/emu_set_layout.cpp."""
import os
import subprocess

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_set_layout(tmp_path):
    exe = str(tmp_path / "emu_set_layout")
    subprocess.check_call(["/usr/bin/g++", "-O2", "-std=c++17", "-Wall", "-o", exe, os.path.join(ROOT, "tests", "emu", "emu_set_layout.cpp")])
    out = subprocess.run([exe], capture_output=True, text=True, timeout=600)
    assert out.returncode == 0, out.stdout + out.stderr
    assert "20000 cases, 0 failures" in out.stdout
