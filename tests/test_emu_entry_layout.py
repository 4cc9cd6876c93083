"""CPU: the entry-layout arithmetic of sk_sketch_set_encode (skani_b200/csrc/entry_layout.cuh) against the host writer's
bytes (put_params + put_sketch, and put_sketch(markers_only(s))) -- entry length and the value at every section offset,
for zero records, all-single and all-multi k-mers, lists of 2 to 1000 positions, zero markers, zero contigs and names of
0 to 17 bytes.  See tests/emu/emu_entry_layout.cpp."""
import os
import subprocess

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_entry_layout(tmp_path):
    exe = str(tmp_path / "emu_entry_layout")
    subprocess.check_call(["/usr/bin/g++", "-O1", "-g", "-std=c++17", "-fsanitize=address", "-fno-omit-frame-pointer", "-o", exe,
                           os.path.join(ROOT, "tests", "emu", "emu_entry_layout.cpp")])
    p = subprocess.run([exe], capture_output=True, text=True, timeout=300, env=dict(os.environ, ASAN_OPTIONS="detect_leaks=0"))
    assert p.returncode == 0 and "48 cases, 0 failures" in p.stdout, p.stdout + p.stderr
