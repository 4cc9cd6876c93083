"""Host emulation of final_kernel's per-item logic (skani_b200/csrc/chain_core.cuh: trim bounds, trimmed mean, population
std, bootstrap replicates and their sequential redo, CI ranks, AF cutoffs, regression gate and GBDT trees) against the
oracle's final_estimate, f32 fields bit for bit, on constructed (est, weight) lists: n around powers of two and the
bootstrap's n >= 10 edge, running weights exactly on the trim bounds, ties, pools below / at / above the guide table,
Lemire rejections, every GBDT node threshold and the cutoff and gate edges.  See tests/emu/emu_final.cpp."""
import os
import re
import subprocess

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_final_estimate_logic_matches_oracle(tmp_path):
    exe = str(tmp_path / "emu_final")
    subprocess.check_call(["/usr/bin/g++", "-O2", "-std=c++17", "-fopenmp", "-ffp-contract=off", "-o", exe,
                           os.path.join(ROOT, "tests", "emu", "emu_final.cpp"), os.path.join(ROOT, "oracle", "skani_oracle.cpp"), "-lz"])
    out = subprocess.run([exe], capture_output=True, text=True, timeout=900)
    assert out.returncode == 0, out.stdout + out.stderr
    assert re.search(r"^0 failures$", out.stdout, re.M), out.stdout
    counts = {}
    for m in re.finditer(r"([a-z0-9 .<>=,-]+?) (\d+)(?=[,;:\n)]| \(|$)", out.stdout):
        counts[m.group(1).strip(" ,;:(")] = int(m.group(2))
    edges = ["estimate kept", "n < 10", "bootstrap", "n a power of two", "not", "search lookups", "lower exact", "lower off by one",
             "upper exact", "upper off by one", "ties", "all 1.0", "below 1024", "at 1024", "above", "rejections",
             "forced redo", "sequential-loop pools", "on a threshold", "next to one", "learned applied", "prediction >= 100",
             "af", "both-af", "ani gate", "bases gate"]
    for e in edges:
        assert counts.get(e, 0) > 0, (e, out.stdout)
